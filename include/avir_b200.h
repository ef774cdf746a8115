// avir_b200.h -- header-only drop-in front-end: avir::CImageResizer<> on NVIDIA H100.
//
// Usage is upstream's (README "Usage Information"): replace `#include "avir.h"` by
// `#include "avir_b200.h"`, link libavirb200.so, and
//
//     avir::CImageResizer<> ImageResizer( 8 );
//     ImageResizer.resizeImage( InBuf, 640, 480, 0, OutBuf, 1024, 768, 3, 0 );
//
// keeps compiling and produces the same bits, computed by hand-written sm_90a kernels.
// Class, member and parameter names follow upstream's public API (avir.h:2262-2547,
// 4569-4685) so that user code is source compatible; the implementation is new: the host
// only plans (avirb200_plan.hpp) and every pixel is produced on the GPU through the C ABI
// in avirb200.h.  There is NO CPU fallback: if libavirb200.so cannot run the call, the
// front-end throws std::runtime_error.
//
// Mirror selection.  Upstream's result bits depend on the `fpclass` template argument
// (summation order, rounding, and even which filter chain is auto-selected), so the
// B200 path declares which upstream fpclass it reproduces:
//     avir::fpclass_def< float >   (default)  -> sequential sums, (int)(v+0.5) rounding
//     avir::fpclass_float4                    -> sequential sums, nearest-even rounding
//     avir::fpclass_float8_dil                -> 8-lane strided sums + hadd, nearest-even
//
// Define AVIRB200_NAMESPACE before including to place everything in another namespace
// (needed only if upstream's avir.h is included in the same translation unit).

#ifndef AVIR_B200_H
#define AVIR_B200_H

#include <charconv>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <string>
#include <tuple>
#include <type_traits>
#include <vector>

#include "avirb200.h"
#include "avirb200_plan.hpp"

#ifndef AVIRB200_NAMESPACE
#define AVIRB200_NAMESPACE avir
#endif

#define AVIR_B200_VERSION "0.1"

namespace AVIRB200_NAMESPACE {

// ---- algorithm parameter sets (upstream avir.h:2262-2464; same field names) ------------

struct CImageResizerParams : public avirb200::plan::Params {
    CImageResizerParams() : avirb200::plan::Params(avirb200::plan::params_preset(0)) {}
    explicit CImageResizerParams(int preset)
        : avirb200::plan::Params(avirb200::plan::params_preset(preset)) {}
};
struct CImageResizerParamsDef : CImageResizerParams { CImageResizerParamsDef() : CImageResizerParams(0) {} };
struct CImageResizerParamsULR : CImageResizerParams { CImageResizerParamsULR() : CImageResizerParams(1) {} };
struct CImageResizerParamsLR : CImageResizerParams { CImageResizerParamsLR() : CImageResizerParams(2) {} };
struct CImageResizerParamsLow : CImageResizerParams { CImageResizerParamsLow() : CImageResizerParams(3) {} };
struct CImageResizerParamsHigh : CImageResizerParams { CImageResizerParamsHigh() : CImageResizerParams(4) {} };
struct CImageResizerParamsUltra : CImageResizerParams { CImageResizerParamsUltra() : CImageResizerParams(5) {} };

// ---- thread pool seam (upstream avir.h:2119-2225) ---------------------------------------
// Accepted for source compatibility; scanlines are scheduled by the GPU, not by this pool.
class CImageResizerThreadPool {
public:
    virtual ~CImageResizerThreadPool() {}
    class CWorkload {
    public:
        virtual ~CWorkload() {}
        virtual void process() = 0;
    };
    virtual int getSuggestedWorkloadCount() const { return 1; }
    virtual void addWorkload(CWorkload* const) {}
    virtual void startAllWorkloads() {}
    virtual void waitAllWorkloadsToFinish() {}
    virtual void removeAllWorkloads() {}
};

// ---- per-call variables (upstream avir.h:2473-2547) --------------------------------------
class CImageResizerVarsBase {
public:
    int ElCount = 0;
    int ElCountIO = 0;
    double k = 0.0; // horizontal step actually used (informational)
    double o = 0.0; // horizontal offset actually used (informational)
    double InGammaMult = 0.0;
    double OutGammaMult = 0.0;
    int BuildModeH = -1; // GPU extension: build modes the planner selected
    int BuildModeV = -1;
};

class CImageResizerVars : public CImageResizerVarsBase {
public:
    double ox = 0.0;
    double oy = 0.0;
    CImageResizerThreadPool* ThreadPool = nullptr;
    bool UseSRGBGamma = false;
    int AlphaIndex = -1;
    int BuildMode = -1;
    int RndSeed = 0;
    void* Stream = nullptr; // GPU extension: cudaStream_t for resizeImageDevice()
};

// GPU extension: tuning / test options applied to every plan a call uses (avirb200_option in
// avirb200.h, indexed by option id; -1 = the plan's default).  None changes a result bit.
struct CImageResizerTuning {
    int opt[6] = {-1, -1, -1, -1, -1, -1};
};

// ---- fpclass tags -------------------------------------------------------------------------
// Tag types naming the upstream processing class to mirror (upstream avir.h:4569-4592,
// avir_float4_sse.h:331, avir_float8_avx.h:370).
struct b200_mirror_def {
    static constexpr avirb200::plan::Mirror mirror() { return avirb200::plan::kMirrorDef; }
    static constexpr int sum_mode = AVIRB200_SUM_INL;
    static constexpr int round_mode = AVIRB200_ROUND_HALFUP_INT;
    static constexpr int id = 0;
    static constexpr int dither = 0;
};
struct b200_mirror_float4 {
    static constexpr avirb200::plan::Mirror mirror() { return avirb200::plan::kMirrorFloat4; }
    static constexpr int sum_mode = AVIRB200_SUM_INL;
    static constexpr int round_mode = AVIRB200_ROUND_RNE_I32;
    static constexpr int id = 1;
    static constexpr int dither = 0;
};
struct b200_mirror_float8_dil {
    static constexpr avirb200::plan::Mirror mirror() { return avirb200::plan::kMirrorFloat8Dil; }
    static constexpr int sum_mode = AVIRB200_SUM_DIL8;
    static constexpr int round_mode = AVIRB200_ROUND_RNE;
    static constexpr int id = 2;
    static constexpr int dither = 0;
};

// Upstream's SIMD value types and ditherer classes, as tags: they only select what the GPU
// path mirrors (avir_float4_sse.h:35, avir_float8_avx.h:36; avir.h:4334, 4442; avir_dil.h:770, 882).
struct float4 {};
struct float8 {};
template <typename fptype> class CImageResizerDithererDefINL {};
template <typename fptype> class CImageResizerDithererErrdINL {};
template <typename fptype, typename fptypesimd> class CImageResizerDithererDefDIL {};
template <typename fptype, typename fptypesimd> class CImageResizerDithererErrdDIL {};

namespace b200_detail {
template <class T> struct mirror_for;      // interleaved classes by their fptype
template <> struct mirror_for<float> { typedef b200_mirror_def type; };
template <> struct mirror_for<float4> { typedef b200_mirror_float4 type; };
template <class D> struct dither_of;       // 0 = per-sample rounding, 1 = error diffusion
template <class T> struct dither_of<CImageResizerDithererDefINL<T> > { static constexpr int value = 0; };
template <class T> struct dither_of<CImageResizerDithererErrdINL<T> > { static constexpr int value = 1; };
template <class T, class S> struct dither_of<CImageResizerDithererDefDIL<T, S> > { static constexpr int value = 0; };
template <class T, class S> struct dither_of<CImageResizerDithererErrdDIL<T, S> > { static constexpr int value = 1; };
} // namespace b200_detail

// avir.h:4569-4592.  afptype float or float4 (the tag above); other types, e.g. double
// intermediates, do not exist on the GPU path.
template <typename afptype = float, typename afptypeatom = afptype,
          class adith = CImageResizerDithererDefINL<afptype> >
class fpclass_def : public b200_detail::mirror_for<afptype>::type {
public:
    static constexpr int dither = b200_detail::dither_of<adith>::value;
};
// avir_dil.h:1000-1023 with float8 (avir_float8_avx.h:370).
template <typename afptype, typename afptypesimd,
          class adith = CImageResizerDithererDefDIL<afptype, afptypesimd> >
class fpclass_def_dil : public b200_mirror_float8_dil {
    static_assert(std::is_same<afptype, float>::value && std::is_same<afptypesimd, float8>::value,
                  "avir_b200: the de-interleaved class mirrored on the GPU path is <float, float8>");
public:
    static constexpr int dither = b200_detail::dither_of<adith>::value;
    // ErrdDIL rounds one scalar at a time: `rsj[0] * TrMulI` converts the float8 constant to
    // float (float8::operator float, avir_float8_avx.h:85), so round() is avir::round<float>,
    // (int)(v + 0.5) (avir_dil.h:958, avir.h:130-135) -- not float8's nearest-even
    static constexpr int round_mode = dither ? AVIRB200_ROUND_HALFUP_INT : AVIRB200_ROUND_RNE;
};
typedef fpclass_def<float4, float> fpclass_float4;
typedef fpclass_def_dil<float, float8> fpclass_float8_dil;

namespace b200_detail {

template <typename T> struct dtype_of;
template <> struct dtype_of<uint8_t> { static constexpr int value = AVIRB200_U8; };
template <> struct dtype_of<uint16_t> { static constexpr int value = AVIRB200_U16; };
template <> struct dtype_of<float> { static constexpr int value = AVIRB200_F32; };
template <> struct dtype_of<double> { static constexpr int value = AVIRB200_F64; };

inline void check(int status, const char* what) {
    if (status == AVIRB200_OK) return;
    if (status == AVIRB200_ERR_ALLOC) throw std::bad_alloc();
    throw std::runtime_error(std::string("avir_b200: ") + what + ": " +
                             avirb200_status_string(status) + " (" + avirb200_last_error() + ")");
}

// Owns an ImagePlan and the C descriptor pointing into it.
struct PlanHolder {
    avirb200::plan::ImagePlan ip;
    avirb200_plan_desc desc;
    avirb200_plan* dev = nullptr;
    int el_count_io = 0;
    ~PlanHolder() { if (dev != nullptr) avirb200_plan_destroy(dev); }
    // the informational outputs of a call (upstream fills them on every call, avir.h:2473-2547)
    void fillVars(CImageResizerVarsBase& v) const {
        v.ElCount = ip.el_count;
        v.ElCountIO = el_count_io;
        v.k = ip.kx; v.o = ip.ox;
        v.InGammaMult = ip.in_gamma_mult;
        v.OutGammaMult = ip.out_gamma_mult;
        v.BuildModeH = ip.h.mode; v.BuildModeV = ip.v.mode;
    }
};

// Process-wide default of the tuning options (what tests and sweeps set through the C driver).
inline CImageResizerTuning& default_tuning() {
    static CImageResizerTuning t;
    return t;
}

inline bool fill_axis(avirb200_axis_desc& ad, const avirb200::plan::AxisPlan& ap, bool dil,
                      bool is_h, int channels) {
    if (ap.unsupported || ap.steps.size() > AVIRB200_MAX_STEPS) return false;
    std::memset(&ad, 0, sizeof(ad));
    ad.src_len = ap.src_len;
    ad.dst_len = ap.dst_len;
    ad.nsteps = static_cast<int32_t>(ap.steps.size());
    for (size_t i = 0; i < ap.steps.size(); ++i) {
        const avirb200::plan::ExecStep& s = ap.steps[i];
        avirb200_step_desc& d = ad.steps[i];
        d.kind = s.kind; d.resample = s.resample; d.latency = s.latency; d.edge = s.edge;
        d.in_len = s.in_len; d.out_len = s.out_len; d.ntaps = s.ntaps; d.order = s.order;
        d.upsampled = s.upsampled; d.skip_odd = s.skip_odd; d.nphases = s.nphases;
        d.out_prefix = s.out_prefix; d.out_suffix = s.out_suffix;
        d.in_prefix = s.in_prefix; d.in_suffix = s.in_suffix;
        d.n_prefix_dc = static_cast<int32_t>(s.prefix_dc.size());
        d.n_suffix_dc = static_cast<int32_t>(s.suffix_dc.size());
        d.taps = s.taps.data();
        d.src_pos = s.src_pos.data(); d.phase = s.phase.data(); d.frac = s.frac.data();
        d.prefix_dc = s.prefix_dc.data(); d.suffix_dc = s.suffix_dc.data();
        // Which accumulators upstream starts from +0 rather than from the first product:
        // every interleaved resize (avir.h:3922-3951, 4006-4036); de-interleaved only the
        // order-1 horizontal multi-channel loop (avir_dil.h:641-652).
        if (s.kind == AVIRB200_STEP_RESIZE)
            d.zero_start = dil ? ((is_h && channels > 1 && s.order == 1) ? 1 : 0) : 1;
    }
    return true;
}

} // namespace b200_detail

// ---- the resizer ----------------------------------------------------------------------------

template <class fpclass = fpclass_def<float> >
class CImageResizer {
public:
    // Same constructor as upstream (avir.h:4630-4639).  Builds the k-independent
    // interpolation bank on the host; touches no GPU state.
    CImageResizer(const int aResBitDepth = 8, const int aSrcBitDepth = 0,
                  const CImageResizerParams& aParams = CImageResizerParamsDef())
        : Params(aParams), ResBitDepth(aResBitDepth),
          SrcBitDepth(aSrcBitDepth == 0 ? aResBitDepth : aSrcBitDepth),
          Designer(new avirb200::plan::Designer(ResBitDepth, SrcBitDepth, aParams,
                                                fpclass::mirror())) {}

    CImageResizer(const CImageResizer&) = delete;
    CImageResizer& operator=(const CImageResizer&) = delete;

    // Upstream signature and semantics (avir.h:4680-4685): host buffers, SrcScanlineSize in
    // elements (<1: SrcWidth*ElCountIO), k = 0 auto / >0 uniform centred / <0 uniform.
    template <typename Tin, typename Tout>
    void resizeImage(const Tin* const SrcBuf, const int SrcWidth, const int SrcHeight,
                     int SrcScanlineSize, Tout* const NewBuf, const int NewWidth,
                     const int NewHeight, const int ElCountIO, const double k,
                     CImageResizerVars* const aVars = nullptr) const {
        if (SrcWidth == 0 || SrcHeight == 0) { // avir.h:4686-4692
            std::memset(NewBuf, 0, (size_t)NewWidth * (size_t)NewHeight * sizeof(Tout));
            return;
        }
        if (NewWidth == 0 || NewHeight == 0) return; // avir.h:4694-4697
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        if (SrcScanlineSize < 1) SrcScanlineSize = SrcWidth * ElCountIO;
        std::shared_ptr<b200_detail::PlanHolder> ph =
            getPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars);
        b200_detail::check(avirb200_resize_host(ph->dev, SrcBuf, (size_t)SrcScanlineSize, NewBuf,
                                                (size_t)NewWidth * ElCountIO),
                           "resizeImage");
    }

    // GPU extension: same call with DEVICE pointers, asynchronous on Vars.Stream.
    // `Workspace` must hold workspaceBytes() bytes of device memory.
    template <typename Tin, typename Tout>
    void resizeImageDevice(const Tin* const dSrcBuf, const int SrcWidth, const int SrcHeight,
                           int SrcScanlineSize, Tout* const dNewBuf, const int NewWidth,
                           const int NewHeight, const int ElCountIO, const double k,
                           void* const Workspace, CImageResizerVars* const aVars = nullptr) const {
        if (SrcWidth == 0 || SrcHeight == 0 || NewWidth == 0 || NewHeight == 0)
            throw std::runtime_error("avir_b200: resizeImageDevice needs non-empty images");
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        if (SrcScanlineSize < 1) SrcScanlineSize = SrcWidth * ElCountIO;
        std::shared_ptr<b200_detail::PlanHolder> ph =
            getPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars);
        b200_detail::check(avirb200_resize_device(ph->dev, dSrcBuf, (size_t)SrcScanlineSize,
                                                  dNewBuf, (size_t)NewWidth * ElCountIO, Workspace,
                                                  Vars.Stream),
                           "resizeImageDevice");
    }

    template <typename Tin, typename Tout>
    size_t workspaceBytes(const int SrcWidth, const int SrcHeight, const int NewWidth,
                          const int NewHeight, const int ElCountIO, const double k,
                          CImageResizerVars* const aVars = nullptr) const {
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        std::shared_ptr<b200_detail::PlanHolder> ph =
            getPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars);
        size_t b = 0;
        b200_detail::check(avirb200_plan_workspace_bytes(ph->dev, &b), "workspaceBytes");
        return b;
    }

    // Host-only: builds (or fetches) the plan descriptor without touching the GPU.
    template <typename Tin, typename Tout>
    std::shared_ptr<b200_detail::PlanHolder>
    buildDescriptor(const int SrcWidth, const int SrcHeight, const int NewWidth,
                    const int NewHeight, const int ElCountIO, const double k,
                    CImageResizerVars& Vars) const {
        using namespace avirb200::plan;
        if (ElCountIO < 1 || ElCountIO > 4)
            throw std::runtime_error("avir_b200: ElCountIO must be 1..4");
        CallDesc c;
        c.src_w = SrcWidth; c.src_h = SrcHeight; c.new_w = NewWidth; c.new_h = NewHeight;
        c.channels = ElCountIO; c.k = k; c.ox = Vars.ox; c.oy = Vars.oy;
        c.in_float = std::is_floating_point<Tin>::value;   // upstream: (Tin)0.25 != 0
        c.out_float = std::is_floating_point<Tout>::value;
        c.in_bytes = (int)sizeof(Tin); c.out_bytes = (int)sizeof(Tout);
        c.use_gamma = Vars.UseSRGBGamma; c.build_mode = Vars.BuildMode;

        std::shared_ptr<b200_detail::PlanHolder> ph(new b200_detail::PlanHolder());
        {
            // The designer's dynamic state (lazily built bank phases) is shared.
            std::lock_guard<std::mutex> lk(Mx);
            ph->ip = plan_image(*Designer, c);
        }
        avirb200_plan_desc& d = ph->desc;
        std::memset(&d, 0, sizeof(d));
        d.src_w = SrcWidth; d.src_h = SrcHeight; d.dst_w = NewWidth; d.dst_h = NewHeight;
        d.channels = ElCountIO;
        d.in_type = b200_detail::dtype_of<Tin>::value;
        d.out_type = b200_detail::dtype_of<Tout>::value;
        d.sum_mode = fpclass::sum_mode;
        d.round_mode = fpclass::round_mode;
        d.dither = c.out_float ? 0 : fpclass::dither; // float output skips dithering (avir.h:5002-5023)
        // Upstream's interleaved float-intermediate class writes float output straight from
        // the column pass and thereby skips applySRGBGamma (avir.h:4956-4979); mirrored.
        // (only when Tout has the intermediate's own size: double output takes the ordinary
        // output stage, avir.h:4956)
        const bool SkipOutGamma = (fpclass::id == 0 && c.out_float && sizeof(Tout) == sizeof(float));
        d.use_gamma = Vars.UseSRGBGamma ? (SkipOutGamma ? 1 : 3) : 0;
        d.alpha_index = (ElCountIO == 4 && (Vars.AlphaIndex == 0 || Vars.AlphaIndex == 3))
                            ? Vars.AlphaIndex : -1;
        d.in_gamma_mult = (float)ph->ip.in_gamma_mult;
        d.out_gamma_mult = (float)ph->ip.out_gamma_mult;
        // Output stage constants (avir.h:5029-5045, 4392-4419).
        d.tr_mul = 1.0f; d.tr_mul_inv = 1.0f; d.pk_out = 0.0f;
        if (!c.out_float) {
            const int range = (sizeof(Tout) == 1 ? 255 : 65535);
            const int trunc = (sizeof(Tout) == 1 ? 8 : 16) - ResBitDepth;
            const double pk = range;
            const double trm = (trunc > 0 ? pk / (range >> trunc) : 1.0);
            d.pk_out = (float)pk;
            d.tr_mul = (float)trm;
            d.tr_mul_inv = (float)(1.0 / trm);
        }
        const bool dil = (fpclass::sum_mode == AVIRB200_SUM_DIL8);
        if (!b200_detail::fill_axis(d.h, ph->ip.h, dil, true, ElCountIO) ||
            !b200_detail::fill_axis(d.v, ph->ip.v, dil, false, ElCountIO))
            throw std::runtime_error("avir_b200: this filtering chain is not available on the "
                                     "GPU path (upsampling factor other than 2)");
        ph->el_count_io = ElCountIO;
        ph->fillVars(Vars);
        return ph;
    }

    // GPU extension: a batch of equally shaped frames on the device (video): one plan, one
    // launch pair per frame, all on Vars.Stream; the frames share `Workspace`.
    template <typename Tin, typename Tout>
    void resizeImageDeviceBatch(const int FrameCount, const Tin* const* const dSrcBufs, const int SrcWidth,
                                const int SrcHeight, int SrcScanlineSize, Tout* const* const dNewBufs,
                                const int NewWidth, const int NewHeight, const int ElCountIO, const double k,
                                void* const Workspace, CImageResizerVars* const aVars = nullptr) const {
        if (SrcWidth == 0 || SrcHeight == 0 || NewWidth == 0 || NewHeight == 0)
            throw std::runtime_error("avir_b200: resizeImageDeviceBatch needs non-empty images");
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        if (SrcScanlineSize < 1) SrcScanlineSize = SrcWidth * ElCountIO;
        std::shared_ptr<b200_detail::PlanHolder> ph =
            getPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars);
        b200_detail::check(avirb200_resize_device_batch(ph->dev, FrameCount,
                                                        reinterpret_cast<const void* const*>(dSrcBufs),
                                                        (size_t)SrcScanlineSize,
                                                        reinterpret_cast<void* const*>(dNewBufs),
                                                        (size_t)NewWidth * ElCountIO, Workspace, Vars.Stream),
                           "resizeImageDeviceBatch");
    }

    // GPU extension: a destination WINDOW -- the pixels [WinX, WinX + WinWidth) x [WinY, WinY + WinHeight)
    // of the NewWidth x NewHeight image resizeImage() makes of the same source, bit-identical to them --
    // computed from the window's source footprint only.  The window is a call argument, not part of the
    // plan: every window of one resize shares its cached plan.  SrcBuf is the WHOLE source image (only the
    // footprint is read); NewBuf receives WinWidth x WinHeight pixels.  Error-diffusion classes throw.
    template <typename Tin, typename Tout>
    void resizeImageWindow(const Tin* const SrcBuf, const int SrcWidth, const int SrcHeight, int SrcScanlineSize,
                           Tout* const NewBuf, const int NewWidth, const int NewHeight, const int ElCountIO,
                           const double k, const int WinX, const int WinY, const int WinWidth, const int WinHeight,
                           CImageResizerVars* const aVars = nullptr) const {
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        if (SrcScanlineSize < 1) SrcScanlineSize = SrcWidth * ElCountIO;
        std::shared_ptr<b200_detail::PlanHolder> ph = getWindowPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight,
                                                                                ElCountIO, k, Vars, "resizeImageWindow");
        b200_detail::check(avirb200_resize_window_host(ph->dev, WinX, WinY, WinWidth, WinHeight, SrcBuf,
                                                       (size_t)SrcScanlineSize, NewBuf, (size_t)WinWidth * ElCountIO),
                           "resizeImageWindow");
    }

    // The same with DEVICE pointers, asynchronous on Vars.Stream: dSrcBuf points at the footprint's first
    // pixel (windowFootprint()) and holds its src_w x src_h pixels, SrcScanlineSize elements apart (< 1:
    // src_w * ElCountIO); `Workspace` holds windowWorkspaceBytes() bytes of device memory.
    template <typename Tin, typename Tout>
    void resizeImageWindowDevice(const Tin* const dSrcBuf, const int SrcWidth, const int SrcHeight,
                                 int SrcScanlineSize, Tout* const dNewBuf, const int NewWidth, const int NewHeight,
                                 const int ElCountIO, const double k, const int WinX, const int WinY,
                                 const int WinWidth, const int WinHeight, void* const Workspace,
                                 CImageResizerVars* const aVars = nullptr) const {
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        std::shared_ptr<b200_detail::PlanHolder> ph = getWindowPlan<Tin, Tout>(
            SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars, "resizeImageWindowDevice");
        avirb200_window_info wi;
        b200_detail::check(avirb200_window_query(ph->dev, WinX, WinY, WinWidth, WinHeight, &wi), "resizeImageWindowDevice");
        if (SrcScanlineSize < 1) SrcScanlineSize = wi.src_w * ElCountIO;
        b200_detail::check(avirb200_resize_window_device(ph->dev, WinX, WinY, WinWidth, WinHeight, dSrcBuf,
                                                         (size_t)SrcScanlineSize, dNewBuf, (size_t)WinWidth * ElCountIO,
                                                         Workspace, Vars.Stream),
                           "resizeImageWindowDevice");
    }

    // The source pixels a window reads (clamped to the image) and the intermediate rows it needs.
    template <typename Tin, typename Tout>
    avirb200_window_info windowFootprint(const int SrcWidth, const int SrcHeight, const int NewWidth,
                                         const int NewHeight, const int ElCountIO, const double k, const int WinX,
                                         const int WinY, const int WinWidth, const int WinHeight,
                                         CImageResizerVars* const aVars = nullptr) const {
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        std::shared_ptr<b200_detail::PlanHolder> ph =
            getWindowPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars, "windowFootprint");
        avirb200_window_info wi;
        b200_detail::check(avirb200_window_query(ph->dev, WinX, WinY, WinWidth, WinHeight, &wi), "windowFootprint");
        return wi;
    }

    template <typename Tin, typename Tout>
    size_t windowWorkspaceBytes(const int SrcWidth, const int SrcHeight, const int NewWidth, const int NewHeight,
                                const int ElCountIO, const double k, const int WinX, const int WinY,
                                const int WinWidth, const int WinHeight, CImageResizerVars* const aVars = nullptr) const {
        CImageResizerVars DefVars;
        CImageResizerVars& Vars = (aVars == nullptr ? DefVars : *aVars);
        std::shared_ptr<b200_detail::PlanHolder> ph = getWindowPlan<Tin, Tout>(
            SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars, "windowWorkspaceBytes");
        size_t b = 0;
        b200_detail::check(avirb200_window_workspace_bytes(ph->dev, WinX, WinY, WinWidth, WinHeight, &b),
                           "windowWorkspaceBytes");
        return b;
    }

    // GPU extension: per-object tuning options (see CImageResizerTuning).
    mutable CImageResizerTuning Tuning;

    // Drops cached plans (device tables and staging buffers).
    void clearPlanCache() const {
        std::lock_guard<std::mutex> lk(Mx);
        Cache.clear();
    }

private:
    typedef std::tuple<int, int, int, int, int, int, int, double, double, double, bool, int, int>
        Key;

    CImageResizerParams Params;
    int ResBitDepth;
    int SrcBitDepth;
    std::unique_ptr<avirb200::plan::Designer> Designer;
    mutable std::mutex Mx;
    mutable std::map<Key, std::shared_ptr<b200_detail::PlanHolder> > Cache;

    template <typename Tin, typename Tout>
    std::shared_ptr<b200_detail::PlanHolder>
    getPlan(const int SrcWidth, const int SrcHeight, const int NewWidth, const int NewHeight,
            const int ElCountIO, const double k, CImageResizerVars& Vars) const {
        const Key key(b200_detail::dtype_of<Tin>::value, b200_detail::dtype_of<Tout>::value,
                      SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars.ox, Vars.oy,
                      Vars.UseSRGBGamma, Vars.AlphaIndex, Vars.BuildMode);
        std::shared_ptr<b200_detail::PlanHolder> ph;
        {
            std::lock_guard<std::mutex> lk(Mx);
            auto it = Cache.find(key);
            if (it != Cache.end()) ph = it->second;
        }
        if (ph) {
            // A cached plan is the plan of the FIRST call with this key.  Upstream re-plans every
            // call, and its build-mode choice reads the filter bank's lazily built phases (avir.h:
            // 4813-4847, 6206-6270), so a repeated identical call may pick another mode there; here a
            // repeated call repeats the first call's bits.  Vars' outputs are refreshed either way.
            ph->fillVars(Vars);
        } else {
            ph = buildDescriptor<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars);
            b200_detail::check(avirb200_plan_create(&ph->desc, &ph->dev), "plan_create");
            std::lock_guard<std::mutex> lk(Mx);
            if (Cache.size() >= 16) Cache.clear(); // bound the device tables held by cached plans
            Cache[key] = ph;
        }
        const CImageResizerTuning& t = b200_detail::default_tuning();
        for (int i = 0; i < 6; ++i) avirb200_plan_set_option(ph->dev, i, Tuning.opt[i] >= 0 ? Tuning.opt[i] : t.opt[i]);
        return ph;
    }

    // The plan of a window call: the whole resize's (windows need non-empty images).
    template <typename Tin, typename Tout>
    std::shared_ptr<b200_detail::PlanHolder>
    getWindowPlan(const int SrcWidth, const int SrcHeight, const int NewWidth, const int NewHeight,
                  const int ElCountIO, const double k, CImageResizerVars& Vars, const char* what) const {
        if (SrcWidth < 1 || SrcHeight < 1 || NewWidth < 1 || NewHeight < 1)
            throw std::runtime_error(std::string("avir_b200: ") + what + " needs non-empty images");
        return getPlan<Tin, Tout>(SrcWidth, SrcHeight, NewWidth, NewHeight, ElCountIO, k, Vars);
    }
};

} // namespace AVIRB200_NAMESPACE

#endif // AVIR_B200_H
