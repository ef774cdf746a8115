// host_capi.cpp -- C entry points over the header-only host side (planner + front-end), so
// that the Python tests and bench.py drive exactly the code a C++ user of
// include/avir_b200.h / include/lancir_b200.h runs.  Built into
// avir_b200/libavirb200_host.so (links libavirb200.so).
//
// This file contains no arithmetic of its own.

#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "avir_b200.h"
#include "lancir_b200.h"

using namespace avirb200::plan;

namespace {

thread_local std::string g_err;

struct CallArgs {
    int mirror, res_bits, src_bits, params_id, tin, tout;
    int sw, sh, nw, nh, ch;
    double k, ox, oy;
    int gamma, alpha, build_mode;
};

void set_vars(avir::CImageResizerVars& v, const CallArgs& a) {
    v.ox = a.ox; v.oy = a.oy;
    v.UseSRGBGamma = (a.gamma != 0);
    v.AlphaIndex = a.alpha;
    v.BuildMode = a.build_mode;
}

// One resizer object per (mirror, bit depths, params): upstream's "one resizer object
// per application" usage (README "Usage Information"), so plan caching is exercised.
template <class fpclass>
avir::CImageResizer<fpclass>& resizer_for(const CallArgs& a) {
    typedef std::tuple<int, int, int> K;
    static std::map<K, std::unique_ptr<avir::CImageResizer<fpclass> > > objs;
    static std::mutex mx;
    std::lock_guard<std::mutex> lk(mx);
    const K key(a.res_bits, a.src_bits, a.params_id);
    auto it = objs.find(key);
    if (it == objs.end())
        it = objs.emplace(key, std::unique_ptr<avir::CImageResizer<fpclass> >(
                                   new avir::CImageResizer<fpclass>(
                                       a.res_bits, a.src_bits,
                                       avir::CImageResizerParams(a.params_id)))).first;
    return *it->second;
}

enum Op { kDesc, kHost, kDevice, kWorkspace, kWinHost, kWinDevice, kWinFootprint, kWinWorkspace };

struct OpArgs {
    Op op;
    const void* src; size_t src_pitch; void* dst; void* workspace; void* stream;
    std::shared_ptr<avir::b200_detail::PlanHolder> holder;
    size_t bytes;
    int mode_h, mode_v;
    int wx, wy, ww, wh;          // window ops: the destination window
    avirb200_window_info info;   // kWinFootprint
};

template <class fpclass, class Tin, class Tout>
void run3(const CallArgs& a, OpArgs& o) {
    avir::CImageResizerVars v;
    set_vars(v, a);
    v.Stream = o.stream;
    if (o.op == kDesc) {
        // A throw-away resizer: descriptor building must not depend on cached state.
        avir::CImageResizer<fpclass> rs(a.res_bits, a.src_bits,
                                        avir::CImageResizerParams(a.params_id));
        o.holder = rs.template buildDescriptor<Tin, Tout>(a.sw, a.sh, a.nw, a.nh, a.ch, a.k, v);
    } else {
        avir::CImageResizer<fpclass>& rs = resizer_for<fpclass>(a);
        if (o.op == kHost)
            rs.resizeImage((const Tin*)o.src, a.sw, a.sh, (int)o.src_pitch, (Tout*)o.dst, a.nw,
                           a.nh, a.ch, a.k, &v);
        else if (o.op == kDevice)
            rs.resizeImageDevice((const Tin*)o.src, a.sw, a.sh, (int)o.src_pitch, (Tout*)o.dst,
                                 a.nw, a.nh, a.ch, a.k, o.workspace, &v);
        else if (o.op == kWinHost)
            rs.resizeImageWindow((const Tin*)o.src, a.sw, a.sh, (int)o.src_pitch, (Tout*)o.dst, a.nw, a.nh, a.ch,
                                 a.k, o.wx, o.wy, o.ww, o.wh, &v);
        else if (o.op == kWinDevice)
            rs.resizeImageWindowDevice((const Tin*)o.src, a.sw, a.sh, (int)o.src_pitch, (Tout*)o.dst, a.nw, a.nh,
                                       a.ch, a.k, o.wx, o.wy, o.ww, o.wh, o.workspace, &v);
        else if (o.op == kWinFootprint)
            o.info = rs.template windowFootprint<Tin, Tout>(a.sw, a.sh, a.nw, a.nh, a.ch, a.k, o.wx, o.wy, o.ww,
                                                             o.wh, &v);
        else if (o.op == kWinWorkspace)
            o.bytes = rs.template windowWorkspaceBytes<Tin, Tout>(a.sw, a.sh, a.nw, a.nh, a.ch, a.k, o.wx, o.wy,
                                                                   o.ww, o.wh, &v);
        else
            o.bytes = rs.template workspaceBytes<Tin, Tout>(a.sw, a.sh, a.nw, a.nh, a.ch, a.k, &v);
    }
    o.mode_h = v.BuildModeH;
    o.mode_v = v.BuildModeV;
}

template <class fpclass, class Tin>
void run2(const CallArgs& a, OpArgs& o) {
    switch (a.tout) {
    case AVIRB200_U8: run3<fpclass, Tin, uint8_t>(a, o); break;
    case AVIRB200_U16: run3<fpclass, Tin, uint16_t>(a, o); break;
    case AVIRB200_F64: run3<fpclass, Tin, double>(a, o); break;
    default: run3<fpclass, Tin, float>(a, o); break;
    }
}

template <class fpclass>
void run1(const CallArgs& a, OpArgs& o) {
    switch (a.tin) {
    case AVIRB200_U8: run2<fpclass, uint8_t>(a, o); break;
    case AVIRB200_U16: run2<fpclass, uint16_t>(a, o); break;
    case AVIRB200_F64: run2<fpclass, double>(a, o); break;
    default: run2<fpclass, float>(a, o); break;
    }
}

int run0(const CallArgs& a, OpArgs& o) {
    if (a.tin < AVIRB200_U8 || a.tin > AVIRB200_F64 || a.tout < AVIRB200_U8 || a.tout > AVIRB200_F64) {
        g_err = "CImageResizer: element type code outside 0..3 (uint8_t, uint16_t, float, double)";
        return -1;
    }
    try {
        switch (a.mirror) {
        case 1: run1<avir::fpclass_float4>(a, o); break;
        case 2: run1<avir::fpclass_float8_dil>(a, o); break;
        // the same three classes with upstream's error-diffusion ditherer
        case 3: run1<avir::fpclass_def<float, float, avir::CImageResizerDithererErrdINL<float> > >(a, o); break;
        case 4: run1<avir::fpclass_def<avir::float4, float, avir::CImageResizerDithererErrdINL<avir::float4> > >(a, o); break;
        case 5: run1<avir::fpclass_def_dil<float, avir::float8, avir::CImageResizerDithererErrdDIL<float, avir::float8> > >(a, o); break;
        default: run1<avir::fpclass_def<float> >(a, o); break;
        }
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
    return 0;
}

void put_axis(std::vector<double>& o, const AxisPlan& a) {
    o.push_back(a.mode);
    o.push_back(a.unsupported ? 1 : 0);
    o.push_back(static_cast<double>(a.steps.size()));
    for (const ExecStep& s : a.steps) {
        const double hd[] = {double(s.kind), double(s.resample), double(s.latency), double(s.edge),
                             double(s.in_len), double(s.out_len), double(s.ntaps), double(s.order),
                             double(s.upsampled), double(s.skip_odd), double(s.nphases),
                             double(s.out_prefix), double(s.out_suffix), double(s.in_prefix),
                             double(s.in_suffix)};
        o.insert(o.end(), hd, hd + 15);
        o.push_back(static_cast<double>(s.taps.size()));
        for (float f : s.taps) o.push_back(f);
        o.push_back(static_cast<double>(s.src_pos.size()));
        for (size_t i = 0; i < s.src_pos.size(); ++i) {
            o.push_back(s.src_pos[i]);
            o.push_back(s.phase[i]);
            o.push_back(s.frac[i]);
        }
    }
}

Mirror mirror_of(int id) {
    switch (id) {
    case 1: case 4: return kMirrorFloat4;
    case 2: case 5: return kMirrorFloat8Dil;
    default: return kMirrorDef;
    }
}

struct DescHandle {
    std::shared_ptr<avir::b200_detail::PlanHolder> holder;
};

} // namespace

extern "C" {

const char* avirb200_host_last_error() { return g_err.c_str(); }

// Test / tuning hook: default plan option of every front-end object in this process
// (avirb200_option ids; value < 0: the plan's own default).
void avirb200_host_set_option(int option, int value) {
    if (option >= 0 && option < 6) avir::b200_detail::default_tuning().opt[option] = value;
}

// Plans the same call twice on one front-end object (no GPU needed: the workspace query only
// plans on a cache miss) and reports the informational Vars outputs of both calls:
// out[0..3] = ElCountIO, k, ... of the first, out[4..7] of the second (cache hit).
int avirb200_host_vars_probe(int sw, int sh, int nw, int nh, double* out) {
    try {
        avir::CImageResizer<avir::fpclass_float4> rs(8);
        for (int i = 0; i < 2; ++i) {
            avir::CImageResizerVars v;
            try {
                rs.workspaceBytes<uint8_t, uint8_t>(sw, sh, nw, nh, 4, 0.0, &v);
            } catch (const std::exception&) {
                // no device: plan_create fails after the descriptor (and Vars) were filled on the
                // first call; the second call then misses the cache as well
            }
            out[4 * i + 0] = v.ElCountIO; out[4 * i + 1] = v.ElCount; out[4 * i + 2] = v.k; out[4 * i + 3] = v.BuildModeH;
        }
    } catch (const std::exception& e) {
        g_err = e.what();
        return -1;
    }
    return 0;
}

// Synthetic input generator of the parity tests and the benchmark (SURVEY.md 8(d)): xorshift32
// from `seed`, one draw per element in memory order, element = (T)((draw & 0xFFFF) * scale) with
// scale 1/257 (u8), 1 (u16), 1/65535 (float), evaluated in double.  dtype: avirb200_dtype.
// Returns the generator's state after the last draw.
uint32_t avirb200_host_fill_xorshift32(void* dst, size_t n, uint32_t seed, int dtype) {
    uint32_t x = seed;
    for (size_t i = 0; i < n; ++i) {
        x ^= x << 13; x ^= x >> 17; x ^= x << 5;
        const double lo = (double)(x & 0xFFFFu);
        if (dtype == AVIRB200_U8) static_cast<uint8_t*>(dst)[i] = (uint8_t)(lo * (1.0 / 257));
        else if (dtype == AVIRB200_U16) static_cast<uint16_t*>(dst)[i] = (uint16_t)lo;
        else static_cast<float*>(dst)[i] = (float)(lo * (1.0 / 65535));
    }
    return x;
}

// Serialises the plan the host would build for one resizeImage() call.
// mirror: 0 def, 1 float4, 2 float8_dil (+3: the same class with the error-diffusion ditherer).  Returns doubles needed (size with cap = 0).
long avirb200_host_plan_dump(int mirror, int res_bits, int src_bits, int params_id, int src_w,
                             int src_h, int new_w, int new_h, int channels, double k, double ox,
                             double oy, int in_float, int out_float, int in_bytes, int out_bytes,
                             int use_gamma, int build_mode, double* out, long cap) {
    Designer d(res_bits, src_bits, params_preset(params_id), mirror_of(mirror));
    CallDesc c{src_w, src_h, new_w, new_h, channels, k, ox, oy, in_float != 0, out_float != 0,
               in_bytes, out_bytes, use_gamma != 0, build_mode};
    const ImagePlan ip = plan_image(d, c);
    std::vector<double> o;
    o.push_back(ip.out_mul);
    o.push_back(ip.in_gamma_mult);
    o.push_back(ip.out_gamma_mult);
    o.push_back(ip.el_count);
    put_axis(o, ip.h);
    put_axis(o, ip.v);
    if (out != nullptr && static_cast<long>(o.size()) <= cap)
        std::memcpy(out, o.data(), o.size() * sizeof(double));
    return static_cast<long>(o.size());
}

// Builds the C-ABI plan descriptor exactly as CImageResizer<>::resizeImage would (no GPU
// needed).  The handle owns the tables the descriptor points to.
void* avirb200_host_desc_create(int mirror, int res_bits, int src_bits, int params_id, int tin,
                                int tout, int sw, int sh, int nw, int nh, int ch, double k,
                                double ox, double oy, int gamma, int alpha, int build_mode,
                                int* modes_out) {
    const CallArgs a{mirror, res_bits, src_bits, params_id, tin, tout, sw, sh, nw, nh, ch,
                     k, ox, oy, gamma, alpha, build_mode};
    OpArgs o{};
    o.op = kDesc;
    if (run0(a, o) != 0) return nullptr;
    if (modes_out != nullptr) { modes_out[0] = o.mode_h; modes_out[1] = o.mode_v; }
    return new DescHandle{o.holder};
}

const avirb200_plan_desc* avirb200_host_desc_get(void* h) {
    return &static_cast<DescHandle*>(h)->holder->desc;
}

void avirb200_host_desc_free(void* h) { delete static_cast<DescHandle*>(h); }

// avir::CImageResizer<fpclass>::resizeImage with host buffers (the drop-in call).
int avirb200_host_resize(int mirror, int res_bits, int src_bits, int params_id, int tin, int tout,
                         const void* src, int sw, int sh, int src_pitch, void* dst, int nw, int nh,
                         int ch, double k, double ox, double oy, int gamma, int alpha,
                         int build_mode) {
    const CallArgs a{mirror, res_bits, src_bits, params_id, tin, tout, sw, sh, nw, nh, ch,
                     k, ox, oy, gamma, alpha, build_mode};
    OpArgs o{};
    o.op = kHost; o.src = src; o.src_pitch = (size_t)src_pitch; o.dst = dst;
    return run0(a, o);
}

// avir::CImageResizer<fpclass>::resizeImageDevice with device buffers.
int avirb200_host_resize_device(int mirror, int res_bits, int src_bits, int params_id, int tin,
                                int tout, const void* d_src, int sw, int sh, int src_pitch,
                                void* d_dst, int nw, int nh, int ch, double k, double ox,
                                double oy, int gamma, int alpha, int build_mode, void* d_workspace,
                                void* stream) {
    const CallArgs a{mirror, res_bits, src_bits, params_id, tin, tout, sw, sh, nw, nh, ch,
                     k, ox, oy, gamma, alpha, build_mode};
    OpArgs o{};
    o.op = kDevice; o.src = d_src; o.src_pitch = (size_t)src_pitch; o.dst = d_dst;
    o.workspace = d_workspace; o.stream = stream;
    return run0(a, o);
}

} // extern "C"

namespace {

// One CLancIR object per thread, as upstream's contract (lancir.h:319-324): the resize and the window
// calls of one geometry share its cached plan.
avir::CLancIR& lancir_obj() {
    thread_local avir::CLancIR obj;
    return obj;
}

template <class Tin, class F>
bool lancir_out(int tout, const void* src, void* dst, F& f) {
    switch (tout) {
    case AVIRB200_U8: f((const Tin*)src, (uint8_t*)dst); return true;
    case AVIRB200_U16: f((const Tin*)src, (uint16_t*)dst); return true;
    case AVIRB200_F32: f((const Tin*)src, (float*)dst); return true;
    case AVIRB200_F64: f((const Tin*)src, (double*)dst); return true;
    case AVIRB200_U32: f((const Tin*)src, (uint32_t*)dst); return true;
    }
    return false;
}

// Calls f((const Tin*)src, (Tout*)dst) with the element types of the codes tin / tout (avirb200_dtype, the
// five CLancIR types); false, without a call, for a code outside 0..4.
template <class F>
bool lancir_types(int tin, int tout, const void* src, void* dst, F f) {
    switch (tin) {
    case AVIRB200_U8: return lancir_out<uint8_t>(tout, src, dst, f);
    case AVIRB200_U16: return lancir_out<uint16_t>(tout, src, dst, f);
    case AVIRB200_F32: return lancir_out<float>(tout, src, dst, f);
    case AVIRB200_F64: return lancir_out<double>(tout, src, dst, f);
    case AVIRB200_U32: return lancir_out<uint32_t>(tout, src, dst, f);
    }
    return false;
}

template <class P> using elem_t = std::remove_const_t<std::remove_pointer_t<P> >;

} // namespace

extern "C" {

// avir::CLancIR::resizeImage with host buffers (lancir_b200.h); returns upstream's return value.
int lancirb200_host_resize(int tin, int tout, const void* src, int sw, int sh, void* dst, int nw,
                           int nh, int ch, int srcssize, int newssize, double kx, double ky,
                           double ox, double oy, double la) {
    avir::CLancIR& obj = lancir_obj();
    avir::CLancIRParams p(srcssize, newssize, kx, ky, ox, oy);
    p.la = la;
    int r = 0;
    if (!lancir_types(tin, tout, src, dst,
                      [&](const auto* s, auto* d) { r = obj.resizeImage(s, sw, sh, d, nw, nh, ch, &p); })) {
        g_err = "lancirb200_host_resize: element type code outside 0..4";
        return -1;
    }
    return r;
}

struct LancirDescHandle {
    avir::CLancIR obj;
    lancirb200_plan_desc desc;
};

// Host-only LANCIR descriptor (the element types select the output-stage constants); null for a type
// code outside 0..4.
void* lancirb200_host_desc_create(int tin, int tout, int sw, int sh, int nw, int nh, int ch,
                                  double kx, double ky, double ox, double oy, double la) {
    LancirDescHandle* h = new LancirDescHandle();
    avir::CLancIRParams p(0, 0, kx, ky, ox, oy);
    p.la = la;
    bool ok = false;
    if (!lancir_types(tin, tout, nullptr, nullptr, [&](const auto* s, auto* d) {
            ok = h->obj.buildDescriptor<elem_t<decltype(s)>, elem_t<decltype(d)> >(h->desc, sw, sh, nw, nh, ch, p);
        }))
        g_err = "lancirb200_host_desc_create: element type code outside 0..4";
    if (!ok) { delete h; return nullptr; }
    return h;
}

// avir::CLancIR::resizeImageWindow (host buffers: the whole source in, the window out),
// resizeImageWindowDevice (src: the window's footprint on the device), windowFootprint and
// windowWorkspaceBytes, on the thread's CLancIR object.  op: 0 host, 1 device, 2 footprint (info: 4 ints,
// lancirb200_window_info), 3 workspace bytes (*bytes).  Returns the method's return value (WinHeight or 0;
// op 3: 1 or 0), -1 for an op or element type code out of range.
int lancirb200_host_window(int op, int tin, int tout, const void* src, int sw, int sh, void* dst, int nw, int nh,
                           int ch, int srcssize, int newssize, double kx, double ky, double ox, double oy,
                           double la, int wx, int wy, int ww, int wh, void* d_workspace, void* stream, int* info,
                           long long* bytes) {
    if (op < 0 || op > 3 || tin < AVIRB200_U8 || tin > AVIRB200_U32 || tout < AVIRB200_U8 || tout > AVIRB200_U32) {
        g_err = "lancirb200_host_window: op outside 0..3 or element type code outside 0..4";
        return -1;
    }
    avir::CLancIR& obj = lancir_obj();
    avir::CLancIRParams p(srcssize, newssize, kx, ky, ox, oy);
    p.la = la;
    lancirb200_window_info wi{};
    size_t nb = 0;
    int r = 0;
    lancir_types(tin, tout, src, dst, [&](const auto* s, auto* d) {
        using TI = elem_t<decltype(s)>;
        using TO = elem_t<decltype(d)>;
        if (op == 0) r = obj.resizeImageWindow(s, sw, sh, d, nw, nh, ch, wx, wy, ww, wh, &p);
        else if (op == 1) r = obj.resizeImageWindowDevice(s, sw, sh, d, nw, nh, ch, wx, wy, ww, wh, d_workspace, stream, &p);
        else if (op == 2) r = obj.windowFootprint<TI, TO>(sw, sh, nw, nh, ch, wx, wy, ww, wh, &wi, &p);
        else r = (nb = obj.windowWorkspaceBytes<TI, TO>(sw, sh, nw, nh, ch, wx, wy, ww, wh, &p)) != 0;
    });
    if (info != nullptr) std::memcpy(info, &wi, sizeof wi);
    if (bytes != nullptr) *bytes = (long long)nb;
    return r;
}

const lancirb200_plan_desc* lancirb200_host_desc_get(void* h) {
    return &static_cast<LancirDescHandle*>(h)->desc;
}

void lancirb200_host_desc_free(void* h) { delete static_cast<LancirDescHandle*>(h); }

long long avirb200_host_workspace_bytes(int mirror, int res_bits, int src_bits, int params_id,
                                        int tin, int tout, int sw, int sh, int nw, int nh, int ch,
                                        double k, double ox, double oy, int gamma, int alpha,
                                        int build_mode) {
    const CallArgs a{mirror, res_bits, src_bits, params_id, tin, tout, sw, sh, nw, nh, ch,
                     k, ox, oy, gamma, alpha, build_mode};
    OpArgs o{};
    o.op = kWorkspace;
    if (run0(a, o) != 0) return -1;
    return (long long)o.bytes;
}

// avir::CImageResizer<fpclass>::resizeImageWindow (host buffers: the whole source in, the window out) and
// resizeImageWindowDevice (d_src: the window's footprint), windowFootprint and windowWorkspaceBytes.
// op: 0 host, 1 device, 2 footprint (info: 6 ints, avirb200_window_info), 3 workspace bytes (*bytes).
int avirb200_host_window(int op, int mirror, int res_bits, int src_bits, int params_id, int tin, int tout,
                         const void* src, int sw, int sh, int src_pitch, void* dst, int nw, int nh, int ch, double k,
                         double ox, double oy, int gamma, int alpha, int build_mode, int wx, int wy, int ww, int wh,
                         void* d_workspace, void* stream, int* info, long long* bytes) {
    const CallArgs a{mirror, res_bits, src_bits, params_id, tin, tout, sw, sh, nw, nh, ch,
                     k, ox, oy, gamma, alpha, build_mode};
    static const Op ops[] = {kWinHost, kWinDevice, kWinFootprint, kWinWorkspace};
    if (op < 0 || op > 3) {
        g_err = "avirb200_host_window: op outside 0..3";
        return -1;
    }
    OpArgs o{};
    o.op = ops[op]; o.src = src; o.src_pitch = (size_t)src_pitch; o.dst = dst;
    o.workspace = d_workspace; o.stream = stream;
    o.wx = wx; o.wy = wy; o.ww = ww; o.wh = wh;
    const int r = run0(a, o);
    if (r == 0 && info != nullptr) std::memcpy(info, &o.info, sizeof o.info);
    if (r == 0 && bytes != nullptr) *bytes = (long long)o.bytes;
    return r;
}

} // extern "C"
