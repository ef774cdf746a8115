// engine.cu -- libavirb200.so: C ABI (include/avirb200.h) over the sm_90a kernels.
//
// Host responsibilities here are strictly device plumbing: copy the planner's tables into
// one device arena, pick tile sizes that fit shared memory, launch the row pass and the
// column pass, move host images for the convenience entry point, and exchange halo rows
// between row-sharded GPUs.  All arithmetic lives in the kernels.
//
// There is no CPU execution path in this library: without a usable CUDA device every
// entry point fails with AVIRB200_ERR_NO_DEVICE / AVIRB200_ERR_CUDA.

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <atomic>
#include <charconv>
#include <condition_variable>
#include <functional>
#include <thread>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "avirb200.h"
#include "device_plan.h"
#include "fast_pass.cuh"
#include "generic_pass.cuh"
#include "host_util.h"
#include "stream_types.h"
#include "stream_launch.h"

using namespace avb;

namespace {
thread_local std::string g_err;
}

int avb::fail(int code, const std::string& msg) {
    g_err = msg;
    return code;
}

namespace {

// The u8 sRGB->linear table: upstream ships 256 float literals (avir.h:234-286) that equal
// the double-precision linearisation formula printed with 7 significant digits.  Regenerated
// here (locale-independent) instead of being copied; tests compare it with the oracle.
void make_srgb_lut(float* lut) {
    for (int i = 0; i < 256; ++i) {
        const double sv = i / 255.0;
        double r;
        if (sv <= 0.04045) {
            r = sv / 12.92;
        } else {
            const double x = (sv + 0.055) / 1.055;
            const double x2 = x * x, x3 = x2 * x, x4 = x2 * x2;
            r = 0.0985766365536824 + 0.839474952656502 * x2 + 0.363287814061725 * x3 -
                0.0125559718896615 / (0.12758338921578 + 0.290283465468235 * x) -
                0.231757513261358 * x - 0.0395365717969074 * x4;
        }
        char buf[64];
        auto res = std::to_chars(buf, buf + sizeof buf, r, std::chars_format::general, 7);
        float f = 0.0f;
        std::from_chars(buf, res.ptr, f);
        lut[i] = f;
    }
}

struct PassConfig {
    int lines_per_block = 0;
    int tile_out = 0;
    int span = 0;
    int pitch = 0;
    size_t smem = 0;
};

struct HostAxis {
    avirb200_axis_desc desc;              // pointers are HOST copies (below)
    std::vector<std::vector<float> > taps, frac, pdc, sdc;
    std::vector<std::vector<int32_t> > src_pos, phase;
    DevAxis dev;                          // device pointers
    DevAxis hostdev;                      // same geometry, host src_pos pointers (range math)
};

} // namespace

namespace {
struct Halo;
}

struct avirb200_plan {
    avirb200_plan_desc desc;     // in_type / out_type: what the KERNELS read and write (F64 -> F32)
    int io_in_type = 0, io_out_type = 0; // the caller's element types
    bool errd = false;                   // integer output through the error-diffusion ditherer
    HostAxis h, v;
    void* arena = nullptr;
    float* d_lut = nullptr;
    int device = 0;
    PassConfig cfg_h, cfg_v;
    FastPlan fast;
    avs::StreamAxisPlan stream_h, stream_v; // chain != 0: the pass runs on the streaming kernel
    // resize_host: the device's shared staging buffers for the duration of a call
    std::mutex mx;
    void* d_src = nullptr;
    void* d_dst = nullptr;
    void* d_ws = nullptr;
    cudaStream_t stream = nullptr;
    // pipelined resize_host: copy-in / copy-out streams and per-band events
    cudaStream_t stream_in = nullptr, stream_out = nullptr;
    std::vector<cudaEvent_t> ev_in, ev_out, ev_d2h, ev_slot; // (+ staged copies of pageable buffers)
    mutable int last_launches = 0;
    // options (avirb200_plan_set_option)
    // 1..3-channel images on the 4-channel kernels (streaming / tile): the source is widened to
    // 4-channel pixels in a scratch copy, both passes run as for RGBA (channels never mix; the
    // pad channel's results are dropped), the destination is narrowed back.  mid_ch: channels of
    // the intermediate (4 then, else the image's).
    bool pad4 = false;
    int mid_ch = 0;
    int opt_family = 0;       // 0 product order, 1 generic kernel only, 2 tile kernel else generic
    int opt_var_h = -1, opt_var_v = -1; // scheduling variant of the streaming passes (-1: default)
    int opt_host_bands = -1;  // resize_host band count (-1: by size)
    int opt_all_chains = 0;
    int opt_overlap = 3;      // sharded: how the halo rows travel (AVIRB200_OPT_OVERLAP_HALO; 3 = fused into the kernels)
    int sm_count = 132;       // of `device`
    Halo* halo = nullptr; // sharded: peer mailboxes (created by the first sharded call)
    cudaStream_t stream_x = nullptr; // sharded: exchange stream
    cudaEvent_t ev_x0 = nullptr, ev_x1 = nullptr;
};

namespace {

int copy_axis_host(HostAxis& ha, const avirb200_axis_desc& ad) {
    if (ad.nsteps < 1 || ad.nsteps > AVIRB200_MAX_STEPS)
        return fail(AVIRB200_ERR_BAD_ARG, "axis: nsteps out of range");
    ha.desc = ad;
    const int n = ad.nsteps;
    ha.taps.resize(n); ha.frac.resize(n); ha.pdc.resize(n); ha.sdc.resize(n);
    ha.src_pos.resize(n); ha.phase.resize(n);
    int prev_len = ad.src_len;
    for (int i = 0; i < n; ++i) {
        const avirb200_step_desc& s = ad.steps[i];
        if (s.in_len != prev_len && !(s.kind == AVIRB200_STEP_RESIZE && s.upsampled))
            return fail(AVIRB200_ERR_BAD_ARG, "axis: step in_len does not chain");
        if (s.kind == AVIRB200_STEP_RESIZE && s.upsampled && s.in_len != prev_len)
            return fail(AVIRB200_ERR_BAD_ARG, "axis: upsampled resize in_len does not chain");
        size_t nt = 0;
        if (s.kind == AVIRB200_STEP_RESIZE) {
            if (s.ntaps < 2 || (s.ntaps & 1) || s.nphases < 1 || s.order < 0 || s.order > 1)
                return fail(AVIRB200_ERR_BAD_ARG, "resize step: bad bank geometry");
            nt = (size_t)s.nphases * s.ntaps * (s.order + 1);
            ha.src_pos[i].assign(s.src_pos, s.src_pos + s.out_len);
            ha.phase[i].assign(s.phase, s.phase + s.out_len);
            ha.frac[i].assign(s.frac, s.frac + s.out_len);
            for (int j = 0; j < s.out_len; ++j) {
                if (s.phase[j] < 0 || s.phase[j] >= s.nphases)
                    return fail(AVIRB200_ERR_BAD_ARG, "resize step: phase index out of range");
                if (j > 0 && s.src_pos[j] < s.src_pos[j - 1])
                    return fail(AVIRB200_ERR_BAD_ARG, "resize step: positions not monotonic");
            }
        } else {
            if (s.ntaps < 1) return fail(AVIRB200_ERR_BAD_ARG, "filter step: no taps");
            if (s.kind == AVIRB200_STEP_FIR && s.resample < 1)
                return fail(AVIRB200_ERR_BAD_ARG, "FIR step: resample < 1");
            nt = (size_t)s.ntaps;
            if (s.kind == AVIRB200_STEP_UPSAMPLE) {
                if (s.resample != 2)
                    return fail(AVIRB200_ERR_UNSUPPORTED, "upsample factor other than 2");
                ha.pdc[i].assign(s.prefix_dc, s.prefix_dc + s.n_prefix_dc);
                ha.sdc[i].assign(s.suffix_dc, s.suffix_dc + s.n_suffix_dc);
            }
        }
        ha.taps[i].assign(s.taps, s.taps + nt);
        prev_len = s.out_len;
    }
    if (prev_len != ad.dst_len) return fail(AVIRB200_ERR_BAD_ARG, "axis: chain does not end at dst_len");
    // from here on the descriptor points at the plan's own copies of the tables
    for (int i = 0; i < n; ++i) {
        avirb200_step_desc& sd = ha.desc.steps[i];
        sd.taps = ha.taps[i].data(); sd.src_pos = ha.src_pos[i].data();
        sd.phase = ha.phase[i].data(); sd.frac = ha.frac[i].data();
        sd.prefix_dc = ha.pdc[i].data(); sd.suffix_dc = ha.sdc[i].data();
    }
    return 0;
}

size_t axis_arena_bytes(const HostAxis& ha) {
    size_t b = 0;
    for (int i = 0; i < ha.desc.nsteps; ++i) {
        b += align_up(ha.taps[i].size() * 4, 256) + align_up(ha.frac[i].size() * 4, 256) +
             align_up(ha.src_pos[i].size() * 4, 256) + align_up(ha.phase[i].size() * 4, 256) +
             align_up(ha.pdc[i].size() * 4, 256) + align_up(ha.sdc[i].size() * 4, 256);
    }
    return b;
}

template <class T>
const T* stage(std::vector<char>& img, size_t& off, char* dbase, const std::vector<T>& v) {
    if (v.empty()) return nullptr;
    const size_t bytes = v.size() * sizeof(T);
    std::memcpy(img.data() + off, v.data(), bytes);
    const T* d = reinterpret_cast<const T*>(dbase + off);
    off += align_up(bytes, 256);
    return d;
}

// The kernels' view of an axis descriptor, with the descriptor's (host) table pointers: what the
// range arithmetic reads.
DevAxis host_axis_view(const avirb200_axis_desc& ad) {
    DevAxis d;
    std::memset(&d, 0, sizeof d);
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

// hostdev: the axis with the plan's host copies of the tables; dev: the same with the copies staged
// into the plan's device arena.
void build_dev_axis(HostAxis& ha, std::vector<char>& img, size_t& off, char* dbase) {
    ha.hostdev = ha.dev = host_axis_view(ha.desc);
    for (int i = 0; i < ha.dev.nsteps; ++i) {
        DevStep& ds = ha.dev.steps[i];
        ds.taps = stage(img, off, dbase, ha.taps[i]);
        ds.src_pos = stage(img, off, dbase, ha.src_pos[i]);
        ds.phase = stage(img, off, dbase, ha.phase[i]);
        ds.frac = stage(img, off, dbase, ha.frac[i]);
        ds.prefix_dc = stage(img, off, dbase, ha.pdc[i]);
        ds.suffix_dc = stage(img, off, dbase, ha.sdc[i]);
    }
}

// Source range a final-output range needs, through the whole chain (host side).
Range chain_source_range(const DevAxis& hd, Range out, int* max_span) {
    Range r = out;
    int span = r.b - r.a + 1;
    for (int i = hd.nsteps - 1; i >= 0; --i) {
        r = step_input_range(hd.steps[i], r, hd.steps[i].src_pos);
        span = imax(span, r.b - r.a + 1);
    }
    if (max_span) *max_span = span;
    return r;
}

const size_t kGenericSmemBudget = 100 * 1024;

PassConfig choose_generic_config(const DevAxis& hd, int channels, int out0, int out1) {
    PassConfig c;
    c.lines_per_block = imax(1, 64 / channels);
    c.pitch = (c.lines_per_block * channels) | 1;
    static const int cand[] = {1024, 768, 512, 384, 256, 192, 128, 96, 64, 48, 32, 24, 16, 12, 8, 4, 2, 1};
    for (int t : cand) {
        int worst = 0;
        for (int j0 = out0; j0 < out1; j0 += t) {
            int sp = 0;
            Range o{j0, imin(j0 + t, out1) - 1};
            chain_source_range(hd, o, &sp);
            worst = imax(worst, sp);
        }
        const size_t smem = 2ull * worst * c.pitch * sizeof(float);
        if (smem <= kGenericSmemBudget || t == 1) {
            c.tile_out = t;
            c.span = worst;
            c.smem = smem;
            break;
        }
    }
    return c;
}

void fill_common(PassParams& p, const avirb200_plan* pl) {
    const avirb200_plan_desc& d = pl->desc;
    p.sum_mode = d.sum_mode;
    p.channels = d.channels;
    p.gamma_in = (d.use_gamma & 1) ? 1 : 0;
    p.gamma_out = (d.use_gamma & 2) ? 1 : 0;
    p.alpha_index = d.alpha_index;
    p.in_gamma_mult = d.in_gamma_mult;
    p.out_gamma_mult = d.out_gamma_mult;
    p.srgb_lut = pl->d_lut;
    p.round_mode = d.round_mode;
    p.tr_mul = d.tr_mul;
    p.tr_mul_inv = d.tr_mul_inv;
    p.pk_out = d.pk_out;
}

int launch_generic(const PassParams& p, const PassConfig& c, cudaStream_t st) {
    dim3 grid((p.out1 - p.out0 + c.tile_out - 1) / c.tile_out,
              (p.n_lines + c.lines_per_block - 1) / c.lines_per_block);
    if (grid.x == 0 || grid.y == 0) return 0;
    if (grid.y > 65535) return fail(AVIRB200_ERR_UNSUPPORTED, "image too large for generic grid");
    if (p.sum_mode == AVIRB200_SUM_DIL8) {
        CUDA_TRY(cudaFuncSetAttribute(generic_pass_kernel<AVIRB200_SUM_DIL8>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem));
        generic_pass_kernel<AVIRB200_SUM_DIL8><<<grid, 256, c.smem, st>>>(p);
    } else {
        CUDA_TRY(cudaFuncSetAttribute(generic_pass_kernel<AVIRB200_SUM_INL>,
                                      cudaFuncAttributeMaxDynamicSharedMemorySize, (int)c.smem));
        generic_pass_kernel<AVIRB200_SUM_INL><<<grid, 256, c.smem, st>>>(p);
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_widen(int type, const void* src, size_t src_pitch, void* dst, int w, int rows, int C, cudaStream_t st);
int launch_narrow(int type, const void* src, void* dst, size_t dst_pitch, int w, int rows, int C, cudaStream_t st);

// 1..3-channel plans whose passes run on the 4-channel kernels in this call (avirb200_plan::pad4)
bool use_pad4(const avirb200_plan* pl) { return pl->pad4 && pl->opt_family != 1; }

// Floats between consecutive intermediate rows, for every kernel family and every band / halo offset.
size_t mid_pitch(const avirb200_plan* pl) { return (size_t)pl->desc.dst_w * pl->mid_ch; }

// Whether a pass runs on the streaming kernel with these buffers (the kernel's source / destination as
// it sees them: a widened plan's scratch copies).  The copies move whole pixels: the row pass's source
// pixels and the column pass's channel pairs must be aligned to their size, the intermediate to 16 bytes.
bool row_pass_on_stream(const avirb200_plan* pl, const void* src, size_t src_pitch, const float* mid) {
    return pl->opt_family == 0 && pl->stream_h.chain != 0 && ((uintptr_t)src % (4 * elem_size(pl->desc.in_type))) == 0 &&
           (src_pitch % 4) == 0 && ((uintptr_t)mid % 16) == 0;
}
bool col_pass_on_stream(const avirb200_plan* pl, const void* dst, size_t dst_pitch, const float* mid) {
    return pl->opt_family == 0 && pl->stream_v.chain != 0 && ((uintptr_t)dst % (2 * elem_size(pl->desc.out_type))) == 0 &&
           (dst_pitch % 2) == 0 && ((uintptr_t)mid % 16) == 0;
}

// Row pass over `rows` source rows (band starting at d_src) into the intermediate band
// starting at d_mid; column pass producing dst rows [out0, out1) from an intermediate
// buffer whose row 0 is global row mid_row_base.
// scratch4: where the band's widened (4-channel) copy goes when use_pad4(pl).
// seg_top / seg_bot (4-channel plans only, the caller checks row_pass_on_stream()): filter only the
// band's first seg_top and last seg_bot rows, in ONE launch.
// xs (sharded calls, fused halo exchange): the band's link, sent through the streaming kernel; *xs_done
// tells whether the streaming kernel took the pass (and so delivered the neighbours' rows).
int run_row_pass(const avirb200_plan* pl, const void* d_src, size_t src_pitch, float* d_mid,
                 int rows, cudaStream_t st, int* launches, void* scratch4 = nullptr, int seg_top = 0, int seg_bot = 0,
                 const avs::StreamLink* xs = nullptr, bool* xs_done = nullptr) {
    if (rows <= 0) return 0;
    // (a non-sticky error another library left in this thread -- NCCL's peer-access probing leaves
    // cudaErrorPeerAccessAlreadyEnabled once the IPC mailboxes have enabled it -- is not this launch's)
    (void)cudaGetLastError();
    const avirb200_plan_desc& d = pl->desc;
    const bool p4 = use_pad4(pl);
    if (p4) {
        if (scratch4 == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "row pass: no scratch for the widened source");
        if (launch_widen(d.in_type, d_src, src_pitch, scratch4, d.src_w, rows, d.channels, st) != 0)
            return fail(AVIRB200_ERR_CUDA, "widening the source failed");
        ++*launches;
        d_src = scratch4;
        src_pitch = (size_t)d.src_w * 4;
    }
    if (row_pass_on_stream(pl, d_src, src_pitch, d_mid)) {
        avs::StreamParams sp;
        avs::stream_fill_row_params(sp, pl->stream_h, d, d_src, (long long)src_pitch, d_mid, (long long)mid_pitch(pl), rows,
                                    pl->d_lut, seg_top, seg_bot);
        if (xs != nullptr) avs::stream_set_sender(sp, *xs);
        const int r = avs::stream_launch(pl->stream_h.chain, false, 0, pl->opt_var_h, sp, pl->sm_count, st);
        if (r == -1) return fail(AVIRB200_ERR_CUDA, "streaming row pass launch failed");
        if (r == 0) { ++*launches; if (xs_done) *xs_done = (xs != nullptr); return 0; }
    }
    if (pl->opt_family != 1 && pl->fast.h_ok) {
        const int r = fast_row_pass(pl->fast, d, d_src, src_pitch, d_mid, mid_pitch(pl), rows, pl->d_lut, pl->sm_count, st);
        if (r == -1) return fail(AVIRB200_ERR_CUDA, "fast row pass launch failed");
        if (r == 0) { ++*launches; return 0; }
    }
    // The generic kernel.  A widened band the 4-channel kernels did not take runs it on the widened
    // copy with 4 channels (the pad channel's results are dropped).
    PassParams p;
    std::memset(&p, 0, sizeof p);
    fill_common(p, pl);
    const PassConfig c = p4 ? choose_generic_config(pl->h.hostdev, 4, 0, d.dst_w) : pl->cfg_h;
    if (p4) p.channels = 4;
    p.ax = pl->h.dev;
    p.is_v = 0;
    p.n_lines = rows;
    p.lines_per_block = c.lines_per_block;
    p.tile_out = c.tile_out;
    p.out0 = 0;
    p.out1 = d.dst_w;
    p.span = c.span;
    p.pitch = c.pitch;
    p.src = d_src;
    p.src_pitch = (long long)src_pitch;
    p.src_type = d.in_type;
    p.dst = d_mid;
    p.dst_pitch = (long long)mid_pitch(pl);
    p.dst_type = AVIRB200_F32;
    ++*launches;
    return launch_generic(p, c, st);
}

// scratch4: where the band's 4-channel destination rows go when use_pad4(pl) (then narrowed into d_dst).
// mid_rows: intermediate rows the buffer holds from mid_row_base on (< 0: up to the image's last row).
// xr (sharded calls, fused halo exchange): the band's link -- the neighbours' rows are read in place from
// its mailbox.  Returns 1, nothing launched, when the streaming kernel cannot take the pass (the caller
// moves the rows into the workspace and calls again without xr).
int run_col_pass(const avirb200_plan* pl, const float* d_mid, int mid_row_base, void* d_dst,
                 size_t dst_pitch, int out0, int out1, cudaStream_t st, int* launches, void* scratch4 = nullptr,
                 int mid_rows = -1, const avs::StreamLink* xr = nullptr) {
    if (out1 <= out0) return 0;
    (void)cudaGetLastError(); // (see run_row_pass)
    const avirb200_plan_desc& d = pl->desc;
    const bool p4 = use_pad4(pl);
    void* const user_dst = d_dst;
    const size_t user_pitch = dst_pitch;
    if (p4) {
        if (scratch4 == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "column pass: no scratch for the 4-channel destination");
        d_dst = scratch4;
        dst_pitch = (size_t)d.dst_w * 4;
    }
    auto finish = [&]() -> int {
        if (!p4) return 0;
        if (launch_narrow(d.out_type, scratch4, user_dst, user_pitch, d.dst_w, out1 - out0, d.channels, st) != 0)
            return fail(AVIRB200_ERR_CUDA, "narrowing the destination failed");
        ++*launches;
        return 0;
    };
    if (col_pass_on_stream(pl, d_dst, dst_pitch, d_mid)) {
        avs::StreamParams sp;
        avs::stream_fill_col_params(sp, pl->stream_v, d, d_mid, (long long)mid_pitch(pl), mid_row_base,
                                    (mid_rows >= 0) ? mid_row_base + mid_rows : d.src_h, d_dst, (long long)dst_pitch,
                                    out0, out1);
        if (xr != nullptr) avs::stream_set_receiver(sp, *xr);
        const int r = avs::stream_launch(pl->stream_v.chain, true, avs::stream_epilogue_code(d), pl->opt_var_v, sp,
                                         pl->sm_count, st);
        if (r == -1) return fail(AVIRB200_ERR_CUDA, "streaming column pass launch failed");
        if (r == 0) { ++*launches; return finish(); }
    }
    if (xr != nullptr) return 1;
    if (pl->opt_family != 1 && pl->fast.v_ok) {
        const int r = fast_col_pass(pl->fast, d, d_mid, mid_pitch(pl), mid_row_base, d_dst, dst_pitch, out0, out1,
                                    pl->d_lut, pl->sm_count, st);
        if (r == -1) return fail(AVIRB200_ERR_CUDA, "fast column pass launch failed");
        if (r == 0) { ++*launches; return finish(); }
    }
    // The generic kernel.  A widened band the tile kernel refused (a shard whose footprint exceeds its
    // shared memory) runs it with 4 channels into the 4-channel scratch, narrowed as after the
    // 4-channel kernels.
    PassParams p;
    std::memset(&p, 0, sizeof p);
    fill_common(p, pl);
    if (p4) p.channels = 4;
    p.ax = pl->v.dev;
    p.is_v = 1;
    p.n_lines = d.dst_w;
    PassConfig c = pl->cfg_v;
    if (p4 || out0 != 0 || out1 != d.dst_h) c = choose_generic_config(pl->v.hostdev, p.channels, out0, out1);
    p.lines_per_block = c.lines_per_block;
    p.tile_out = c.tile_out;
    p.out0 = out0;
    p.out1 = out1;
    p.span = c.span;
    p.pitch = c.pitch;
    p.src = d_mid;
    p.src_pitch = (long long)mid_pitch(pl);
    p.src_type = AVIRB200_F32;
    p.src_row_base = mid_row_base;
    p.dst = d_dst;
    p.dst_pitch = (long long)dst_pitch;
    p.dst_type = d.out_type;
    p.dst_row_base = out0;
    ++*launches;
    const int r = launch_generic(p, c, st);
    return r != 0 ? r : finish();
}

// ---- NCCL through dlopen (no link-time dependency) -------------------------------------------

struct Id128 { char b[128]; }; // ncclUniqueId (passed by value)

struct Nccl {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, Id128, int) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*Send)(const void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};

Nccl* nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, []() {
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) {
            n.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (n.lib) break;
        }
        if (!n.lib) return;
        n.GetUniqueId = (int (*)(void*))dlsym(n.lib, "ncclGetUniqueId");
        n.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(n.lib, "ncclCommInitRank");
        n.CommDestroy = (int (*)(void*))dlsym(n.lib, "ncclCommDestroy");
        n.Send = (int (*)(const void*, size_t, int, int, void*, cudaStream_t))dlsym(n.lib, "ncclSend");
        n.Recv = (int (*)(void*, size_t, int, int, void*, cudaStream_t))dlsym(n.lib, "ncclRecv");
        n.GroupStart = (int (*)())dlsym(n.lib, "ncclGroupStart");
        n.GroupEnd = (int (*)())dlsym(n.lib, "ncclGroupEnd");
        n.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(n.lib, "ncclAllGather");
        n.GetErrorString = (const char* (*)(int))dlsym(n.lib, "ncclGetErrorString");
    });
    if (!n.lib || !n.GetUniqueId || !n.CommInitRank || !n.Send || !n.Recv || !n.GroupStart ||
        !n.GroupEnd)
        return nullptr;
    return &n;
}

#define NCCL_TRY(expr)                                                                  \
    do {                                                                                \
        int r_ = (expr);                                                                \
        if (r_ != 0)                                                                    \
            return fail(AVIRB200_ERR_NCCL, std::string(#expr) + ": " +                  \
                                               (nc->GetErrorString ? nc->GetErrorString(r_) \
                                                                   : "nccl error"));     \
    } while (0)

int shard_compute_axis(const DevAxis& vaxis, int rank, int nranks, avirb200_shard_info* info) {
    if (nranks < 1 || rank < 0 || rank >= nranks) return fail(AVIRB200_ERR_BAD_ARG, "bad rank");
    const int src_h = vaxis.src_len, dst_h = vaxis.dst_len;
    auto src_split = [&](int r) { return (int)((long long)src_h * r / nranks); };
    auto dst_split = [&](int r) { return (int)((long long)dst_h * r / nranks); };
    info->src_row0 = src_split(rank);
    info->src_rows = src_split(rank + 1) - info->src_row0;
    info->dst_row0 = dst_split(rank);
    info->dst_rows = dst_split(rank + 1) - info->dst_row0;
    if (info->dst_rows <= 0 || info->src_rows <= 0)
        return fail(AVIRB200_ERR_UNSUPPORTED, "image has fewer rows than ranks");
    Range need = chain_source_range(vaxis,
                                    Range{info->dst_row0, info->dst_row0 + info->dst_rows - 1},
                                    nullptr);
    // The band always contains the rank's own rows (they are produced locally anyway).
    need.a = imin(need.a, info->src_row0);
    need.b = imax(need.b, info->src_row0 + info->src_rows - 1);
    info->need_row0 = need.a;
    info->need_rows = need.b - need.a + 1;
    info->halo_up = info->src_row0 - need.a;
    info->halo_down = need.b - (info->src_row0 + info->src_rows - 1);
    if (rank > 0 && info->halo_up > src_split(rank) - src_split(rank - 1))
        return fail(AVIRB200_ERR_UNSUPPORTED, "halo exceeds the neighbouring band (too many ranks)");
    if (rank + 1 < nranks && info->halo_down > src_split(rank + 2 > nranks ? nranks : rank + 2) -
                                                   src_split(rank + 1))
        return fail(AVIRB200_ERR_UNSUPPORTED, "halo exceeds the neighbouring band (too many ranks)");
    return 0;
}

int shard_compute(const avirb200_plan* pl, int rank, int nranks, avirb200_shard_info* info) {
    return shard_compute_axis(pl->v.hostdev, rank, nranks, info);
}

// ---- error-diffusion ditherer (upstream CImageResizerDithererErrdINL / ErrdDIL) ---------------
// avir.h:4485-4525, avir_dil.h:927-986, driven row by row from resizeImage (avir.h:5046-5064).
// Per channel, pixel j of row y:   R = (v[j] + D_y[j]) [+ 0.364842 * Noise(j-1)];
//   z = round(R * TrMulI) * TrMul;  Noise = R - z;  out = clamp(z, 0, PkOut);
// and the row below adds D_{y+1}[q] = ((0 + 0.063011*Noise(q-1)) + 0.364842*Noise(q)) + 0.207305*Noise(q+1)
// (the order in which upstream's three "+=" reach the element).  The recursion runs along the
// row AND down the rows, so the parallel form is a wavefront: row y+1 may process pixel q once
// row y has finished pixel q+1.  One warp takes 32 consecutive rows as a systolic array -- lane =
// row, lane l works on pixel t - 2l at step t and hands D_{y+1}[q] to lane l+1 by shuffle, one
// step before it is needed; lane 31 hands its values to lane 0 of the next warp (another block)
// through a row of boundary values in global memory plus a progress counter.  Every block is
// resident at once (one warp each); a block only ever waits for the block before it.
// Quirk kept: the de-interleaved class stores a row as consecutive channel planes and runs them
// one after the other, so the "Dith[j-1] +=" of pixel 0 of plane c+1 lands on the last pixel of
// plane c (avir_dil.h:964, rsdj[-1] with j = 0):  D_{y+1}[c][W-1] gains + 0.207305*Noise_{c+1}(0).
struct ErrdParams {
    const float* src;     // [H][W*C] gamma-corrected floats (the column pass's output)
    void* dst;
    long long dst_pitch;  // elements
    int W, H, dst_type, round_mode;
    int planar;           // de-interleaved class: channel c+1's pixel 0 also feeds channel c's last D (see below)
    float tr_mul, tr_mul_inv, pk_out;
    float* boundary;      // [groups][W*C]
    int* progress;        // [groups]: pixels of the group's last row whose D values are published
};

template <int C>
__global__ void __launch_bounds__(32) errd_kernel(const __grid_constant__ ErrdParams p) {
    const int g = blockIdx.x, lane = threadIdx.x;
    const int W = p.W, y = g * 32 + lane;
    const bool rowok = y < p.H;
    const float* row = p.src + (size_t)(rowok ? y : p.H - 1) * W * C;
    const float* bnd_in = p.boundary + (size_t)(g > 0 ? g - 1 : 0) * W * C;
    float* bnd_out = p.boundary + (size_t)g * W * C;
    volatile int* prog_in = p.progress + (g > 0 ? g - 1 : 0);
    volatile int* prog_out = p.progress + g;
    const bool publish = (lane == 31) && ((g + 1) * 32 < p.H);
    int seen = 0; // lane 0: pixels the group above is known to have published
    float nm1[C], c3p[C], part[C], dn[C], v[C], vn[C], n2first[C];
#pragma unroll
    for (int c = 0; c < C; ++c) { nm1[c] = c3p[c] = part[c] = dn[c] = n2first[c] = 0.0f; v[c] = vn[c] = 0.0f; }
    if (lane == 0 && W > 0) {
#pragma unroll
        for (int c = 0; c < C; ++c) vn[c] = __ldg(row + c);
    }
    const int steps = W + 2 * 31 + 1;
    for (int t = 0; t < steps; ++t) {
        const int pix = t - 2 * lane;
        const bool on = rowok && pix >= 0 && pix < W;
        // D of this pixel: from the lane above (finalised there during the previous step) ...
        float din[C];
#pragma unroll
        for (int c = 0; c < C; ++c) din[c] = __shfl_up_sync(0xffffffffu, dn[c], 1);
        // ... or, for the group's first row, from the group above (row 0 of the image: zero)
        if (lane == 0 && on) {
            if (g == 0) {
#pragma unroll
                for (int c = 0; c < C; ++c) din[c] = 0.0f;
            } else {
                while (seen <= pix) seen = *prog_in;
                __threadfence();
#pragma unroll
                for (int c = 0; c < C; ++c) din[c] = __ldcg(bnd_in + (size_t)pix * C + c);
            }
        }
#pragma unroll
        for (int c = 0; c < C; ++c) v[c] = vn[c];
        // the next pixel's input does not depend on the recursion: fetch it now
        if (rowok && pix + 1 >= 0 && pix + 1 < W) {
#pragma unroll
            for (int c = 0; c < C; ++c) vn[c] = __ldg(row + (size_t)(pix + 1) * C + c);
        }
        if (on) {
            float o[C];
#pragma unroll
            for (int c = 0; c < C; ++c) {
                float R = __fadd_rn(v[c], din[c]);
                if (pix > 0) R = __fadd_rn(R, nm1[c]);
                const float z0 = __fmul_rn(avb::round_out(__fmul_rn(R, p.tr_mul_inv), p.round_mode), p.tr_mul);
                const float noise = __fsub_rn(R, z0);
                o[c] = z0 < 0.0f ? 0.0f : (z0 > p.pk_out ? p.pk_out : z0);
                const float n1 = __fmul_rn(noise, 0.364842f);
                const float n2 = __fmul_rn(noise, 0.207305f);
                const float n3 = __fmul_rn(noise, 0.063011f);
                if (pix == 0) n2first[c] = n2;
                dn[c] = __fadd_rn(part[c], n2); // D_{y+1}[pix-1] is complete (unused for pix == 0)
                part[c] = (pix == 0) ? __fadd_rn(0.0f, n1) : __fadd_rn(__fadd_rn(0.0f, c3p[c]), n1);
                c3p[c] = n3;
                nm1[c] = n1;
            }
            const size_t oi = (size_t)y * (size_t)p.dst_pitch + (size_t)pix * C;
            if (p.dst_type == AVIRB200_U8) {
#pragma unroll
                for (int c = 0; c < C; ++c) static_cast<unsigned char*>(p.dst)[oi + c] = (unsigned char)o[c];
            } else {
#pragma unroll
                for (int c = 0; c < C; ++c) static_cast<unsigned short*>(p.dst)[oi + c] = (unsigned short)o[c];
            }
        } else if (rowok && pix == W) {
#pragma unroll
            for (int c = 0; c < C; ++c) {
                dn[c] = part[c]; // D_{y+1}[W-1]: no pixel to its right ...
                if (p.planar && c + 1 < C) dn[c] = __fadd_rn(dn[c], n2first[c + 1]); // ... but the next plane's pixel 0
            }
        }
        if (publish) {
            const int q = (on && pix >= 1) ? pix - 1 : ((pix == W) ? W - 1 : -1);
            if (q >= 0) {
#pragma unroll
                for (int c = 0; c < C; ++c) __stcg(bnd_out + (size_t)q * C + c, dn[c]);
                __threadfence();
                *prog_out = q + 1;
            }
        }
    }
}

// ---- 1..3-channel images on the 4-channel kernels: widen the source, narrow the destination ----
template <typename T>
__global__ void __launch_bounds__(256) widen_channels_kernel(const T* __restrict__ src, long long src_pitch,
                                                             T* __restrict__ dst, int w, int rows, int C) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= (long long)w * rows) return;
    const int y = (int)(i / w), x = (int)(i - (long long)y * w);
    const T* s = src + (long long)y * src_pitch + (long long)x * C;
    T v[4] = {T(0), T(0), T(0), T(0)};
    for (int c = 0; c < C; ++c) v[c] = s[c];
    T* o = dst + i * 4;
    o[0] = v[0]; o[1] = v[1]; o[2] = v[2]; o[3] = v[3];
}

template <typename T>
__global__ void __launch_bounds__(256) narrow_channels_kernel(const T* __restrict__ src, T* __restrict__ dst,
                                                              long long dst_pitch, int w, int rows, int C) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= (long long)w * rows) return;
    const int y = (int)(i / w), x = (int)(i - (long long)y * w);
    const T* s = src + i * 4;
    T* o = dst + (long long)y * dst_pitch + (long long)x * C;
    for (int c = 0; c < C; ++c) o[c] = s[c];
}

int launch_widen(int type, const void* src, size_t src_pitch, void* dst, int w, int rows, int C, cudaStream_t st) {
    const long long n = (long long)w * rows;
    const unsigned g = (unsigned)((n + 255) / 256);
    if (type == AVIRB200_U8)
        widen_channels_kernel<unsigned char><<<g, 256, 0, st>>>((const unsigned char*)src, (long long)src_pitch, (unsigned char*)dst, w, rows, C);
    else if (type == AVIRB200_U16)
        widen_channels_kernel<unsigned short><<<g, 256, 0, st>>>((const unsigned short*)src, (long long)src_pitch, (unsigned short*)dst, w, rows, C);
    else
        widen_channels_kernel<float><<<g, 256, 0, st>>>((const float*)src, (long long)src_pitch, (float*)dst, w, rows, C);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

int launch_narrow(int type, const void* src, void* dst, size_t dst_pitch, int w, int rows, int C, cudaStream_t st) {
    const long long n = (long long)w * rows;
    const unsigned g = (unsigned)((n + 255) / 256);
    if (type == AVIRB200_U8)
        narrow_channels_kernel<unsigned char><<<g, 256, 0, st>>>((const unsigned char*)src, (unsigned char*)dst, (long long)dst_pitch, w, rows, C);
    else if (type == AVIRB200_U16)
        narrow_channels_kernel<unsigned short><<<g, 256, 0, st>>>((const unsigned short*)src, (unsigned short*)dst, (long long)dst_pitch, w, rows, C);
    else
        narrow_channels_kernel<float><<<g, 256, 0, st>>>((const float*)src, (float*)dst, (long long)dst_pitch, w, rows, C);
    return cudaGetLastError() == cudaSuccess ? 0 : -1;
}

// ---- double image buffers: the casts upstream's pack / unpack perform, as two small kernels ----

__global__ void __launch_bounds__(256) narrow_f64_kernel(const double* __restrict__ src, long long src_pitch,
                                                        float* __restrict__ dst, int row_elems, int rows) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long n = (long long)row_elems * rows;
    if (i >= n) return;
    const int y = (int)(i / row_elems), x = (int)(i - (long long)y * row_elems);
    dst[i] = __double2float_rn(src[(long long)y * src_pitch + x]); // (fptypeatom) ip[c], avir.h:2803-2806
}

__global__ void __launch_bounds__(256) widen_f32_kernel(const float* __restrict__ src, double* __restrict__ dst,
                                                       long long dst_pitch, int row_elems, int rows) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long n = (long long)row_elems * rows;
    if (i >= n) return;
    const int y = (int)(i / row_elems), x = (int)(i - (long long)y * row_elems);
    dst[(long long)y * dst_pitch + x] = (double)src[i]; // (Tout) v[c], avir.h:3168-3171
}

// error diffusion: per 32-row group one row of boundary values + one progress counter
int errd_groups(const avirb200_plan* pl) { return (pl->desc.dst_h + 31) / 32; }

// The workspace of one call: byte offsets of its segments, in this order, each 256-byte aligned.
//   mid        the intermediate: mid_rows rows of mid_pitch() floats (at offset 0)
//   in32       float copy of a double source                                  } whole-image calls only
//   out32      float copy of the destination (double output, error diffusion) } (resize_device):
//   errd_bnd   error diffusion: boundary rows, one per 32-row group           } sharded and per-pass
//   errd_prog  error diffusion: progress counters                             } calls refuse such plans
//   src4       the widened source of src_rows rows   } widened plans (pad4) only
//   dst4       the widened destination of dst_rows rows }
// Segments a plan does not use are empty.
struct WsLayout {
    size_t in32, out32, errd_bnd, errd_prog, src4, dst4, total;
};
WsLayout ws_layout(const avirb200_plan* pl, int mid_rows, int src_rows, int dst_rows, bool whole) {
    const avirb200_plan_desc& d = pl->desc;
    const bool f64_in = whole && pl->io_in_type == AVIRB200_F64;
    const bool f32_out = whole && (pl->io_out_type == AVIRB200_F64 || pl->errd);
    const bool errd = whole && pl->errd;
    WsLayout w;
    size_t off = align_up((size_t)mid_rows * mid_pitch(pl) * sizeof(float), 256);
    auto seg = [&](bool on, size_t bytes) {
        const size_t at = off;
        if (on) off += align_up(bytes, 256);
        return at;
    };
    w.in32 = seg(f64_in, (size_t)d.src_w * d.src_h * d.channels * sizeof(float));
    w.out32 = seg(f32_out, (size_t)d.dst_w * d.dst_h * d.channels * sizeof(float));
    w.errd_bnd = seg(errd, (size_t)errd_groups(pl) * d.dst_w * d.channels * sizeof(float));
    w.errd_prog = seg(errd, (size_t)errd_groups(pl) * sizeof(int));
    w.src4 = seg(pl->pad4, (size_t)src_rows * d.src_w * 4 * elem_size(d.in_type));
    w.dst4 = seg(pl->pad4, (size_t)dst_rows * d.dst_w * 4 * elem_size(d.out_type));
    w.total = off;
    return w;
}
// The whole image's layout (resize_device, the per-pass entry points, the banded host call).
WsLayout ws_layout(const avirb200_plan* pl) { return ws_layout(pl, pl->desc.src_h, pl->desc.src_h, pl->desc.dst_h, true); }
// One band of the sharded schedule.
WsLayout ws_layout(const avirb200_plan* pl, const avirb200_shard_info& si) {
    return ws_layout(pl, si.need_rows, si.src_rows, si.dst_rows, false);
}

// ---- host-call staging: one set of device buffers per device, shared by every plan ----------------
// (a front-end object caches up to 16 plans; per-plan staging of 8K frames would hold ~1 GB each)
struct Staging {
    std::mutex mx; // held for the whole host call: host calls on one device run one at a time
    void *d_src = nullptr, *d_dst = nullptr, *d_ws = nullptr;
    size_t src_b = 0, dst_b = 0, ws_b = 0;
    // page-locked bounce buffers for callers' pageable (malloc) images: a ring of source bands
    // and the whole destination
    char *h_in = nullptr, *h_out = nullptr;
    size_t h_in_b = 0, h_out_b = 0;
};

// A few host threads that move image rows between the caller's pageable memory and the
// page-locked bounce buffers (one thread's memcpy is slower than PCIe).
class CopyPool {
public:
    static CopyPool& get() {
        // never destroyed: its detached workers wait on the condition variable for the life of the
        // process, and destroying a condition variable with waiters blocks (process exit would hang)
        static CopyPool* p = new CopyPool();
        return *p;
    }
    // rows of `row_bytes` from src (pitch sp) to dst (pitch dp), split over the workers and the caller
    void copy2d(char* dst, size_t dp, const char* src, size_t sp, size_t row_bytes, int rows) {
        if (rows <= 0) return;
        const int parts = (int)std::min<size_t>(nthreads_ + 1, std::max<size_t>(1, (size_t)rows * row_bytes >> 20));
        if (parts <= 1) { rows_copy(dst, dp, src, sp, row_bytes, 0, rows); return; }
        // (completion state outlives this call: a worker may still be leaving its critical section
        // when the caller has already seen the count reach zero)
        struct Done {
            std::mutex m;
            std::condition_variable cv;
            int left;
        };
        std::shared_ptr<Done> done(new Done());
        done->left = parts - 1;
        for (int i = 1; i < parts; ++i) {
            const int a = (int)((long long)rows * i / parts), b = (int)((long long)rows * (i + 1) / parts);
            submit([=] {
                rows_copy(dst, dp, src, sp, row_bytes, a, b);
                std::lock_guard<std::mutex> g(done->m);
                if (--done->left == 0) done->cv.notify_one();
            });
        }
        rows_copy(dst, dp, src, sp, row_bytes, 0, (int)((long long)rows / parts));
        std::unique_lock<std::mutex> g(done->m);
        done->cv.wait(g, [&] { return done->left == 0; });
    }

private:
    CopyPool() {
        unsigned hw = std::thread::hardware_concurrency();
        nthreads_ = hw >= 32 ? 7 : (hw >= 8 ? 3 : 1);
        for (size_t i = 0; i < nthreads_; ++i) std::thread([this] { run(); }).detach();
    }
    static void rows_copy(char* dst, size_t dp, const char* src, size_t sp, size_t row_bytes, int a, int b) {
        if (dp == row_bytes && sp == row_bytes) { std::memcpy(dst + (size_t)a * dp, src + (size_t)a * sp, (size_t)(b - a) * row_bytes); return; }
        for (int y = a; y < b; ++y) std::memcpy(dst + (size_t)y * dp, src + (size_t)y * sp, row_bytes);
    }
    void submit(std::function<void()> f) {
        { std::lock_guard<std::mutex> g(m_); q_.push_back(std::move(f)); }
        cv_.notify_one();
    }
    void run() {
        for (;;) {
            std::function<void()> f;
            {
                std::unique_lock<std::mutex> g(m_);
                cv_.wait(g, [&] { return !q_.empty(); });
                f = std::move(q_.front());
                q_.erase(q_.begin());
            }
            f();
        }
    }
    size_t nthreads_ = 1;
    std::mutex m_;
    std::condition_variable cv_;
    std::vector<std::function<void()> > q_;
};

bool is_pageable(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
int grow_host(char** p, size_t* have, size_t need) {
    if (*have >= need) return 0;
    if (*p) cudaFreeHost(*p);
    *p = nullptr; *have = 0;
    CUDA_TRY(cudaHostAlloc(reinterpret_cast<void**>(p), need, cudaHostAllocDefault));
    *have = need;
    return 0;
}
Staging& staging_of(int device) {
    static Staging pool[64];
    return pool[(unsigned)device & 63u];
}
int grow(void** p, size_t* have, size_t need) {
    if (*have >= need) return 0;
    cudaFree(*p);
    *p = nullptr; *have = 0;
    CUDA_TRY(cudaMalloc(p, need));
    *have = need;
    return 0;
}
// Points the plan's d_src / d_dst / d_ws at the device's staging buffers (grown to the sizes
// asked for).  The caller holds staging_of(pl->device).mx.
int plan_staging(avirb200_plan* pl, size_t in_bytes, size_t out_bytes, size_t ws) {
    Staging& sg = staging_of(pl->device);
    int r;
    if ((r = grow(&sg.d_src, &sg.src_b, in_bytes)) != 0 || (r = grow(&sg.d_dst, &sg.dst_b, out_bytes)) != 0 ||
        (r = grow(&sg.d_ws, &sg.ws_b, ws)) != 0)
        return r;
    pl->d_src = sg.d_src; pl->d_dst = sg.d_dst; pl->d_ws = sg.d_ws;
    return 0;
}

// ---- sharded calls: peer mailboxes for the halo rows ------------------------------------------------
// NCCL's send/recv between the two passes costs a kernel launch on every rank and runs on SMs the
// persistent pass kernels want.  Instead every rank owns a MAILBOX in device memory that its two
// neighbours map through CUDA IPC (handles all-gathered over the caller's communicator once per
// plan): a rank filters the rows its neighbours need FIRST, pushes them with the copy engines
// (peer copy over NVLink, no SM) into the neighbours' mailboxes followed by a sequence number,
// and filters its interior rows meanwhile; before the column pass a one-warp kernel waits for
// the neighbours' sequence numbers and the rows move from the mailbox into the workspace.
// Two slots (call parity): a rank can be at most one call ahead of a neighbour, because its
// column pass needs that neighbour's rows of the same call.  avirb200_resize_sharded_local keeps
// one mailbox per band in one device's memory, with one slot.
//
// The mailbox of band q, as MailboxLayout describes it:
//   [256 B header: flag "from above" at +0, flag "from below" at +4, the sender's counters at +64]
//   slot 0: [rows from q-1: halo_up(q)] [rows from q+1: halo_down(q), at +align256(up_bytes)]   slot 1: the same
struct MailboxLayout {
    static constexpr size_t kHeader = 256, kCounters = 64;
    size_t up_bytes = 0, down_bytes = 0;
    MailboxLayout() = default;
    MailboxLayout(const avirb200_plan* pl, const avirb200_shard_info& si)
        : up_bytes((size_t)si.halo_up * mid_pitch(pl) * sizeof(float)),
          down_bytes((size_t)si.halo_down * mid_pitch(pl) * sizeof(float)) {}
    size_t slot_bytes() const { return align_up(up_bytes, 256) + align_up(down_bytes, 256); }
    size_t bytes(int slots) const { return kHeader + (size_t)slots * slot_bytes(); }
    // the mailbox at `box` (this process's address of it), slot `slot`
    avs::StreamMailbox at(char* box, int slot) const {
        char* s = box + kHeader + (size_t)slot * slot_bytes();
        return {reinterpret_cast<float*>(s), reinterpret_cast<float*>(s + align_up(up_bytes, 256)),
                reinterpret_cast<unsigned*>(box), reinterpret_cast<unsigned long long*>(box + kCounters)};
    }
};

struct Halo {
    void* comm = nullptr;
    int rank = -1, nranks = 0;
    bool usable = false;
    char* box = nullptr;       // my mailbox
    char* box_up = nullptr;    // rank-1's mailbox, mapped
    char* box_down = nullptr;  // rank+1's mailbox, mapped
    MailboxLayout mine, above, below; // the layouts of the three
    unsigned long long off_up = 0, off_down = 0; // the neighbours' mailboxes inside their allocations
    unsigned seq = 0;
    unsigned* h_seq = nullptr; // pinned ring of sequence numbers the flag copies read
};

// Waits for the neighbours' sequence numbers, then moves their rows from the mailbox into the
// workspace (both directions, one launch).
__global__ void __launch_bounds__(256) halo_pull_kernel(const volatile unsigned* flags, unsigned seq, int need_up,
                                                        int need_down, const float4* up_src, float4* up_dst, size_t up_n,
                                                        const float4* down_src, float4* down_dst, size_t down_n) {
    if (threadIdx.x < 2) {
        const int t = threadIdx.x;
        if ((t == 0 && need_up) || (t == 1 && need_down)) {
            long long spins = 0;
            while ((int)(flags[t] - seq) < 0) {
                if (++spins > (1ll << 31)) __trap(); // a neighbour never delivered: fail instead of hanging
                __nanosleep(100);
            }
            __threadfence_system();
        }
    }
    __syncthreads();
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < up_n; i += stride) up_dst[i] = __ldcv(up_src + i);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < down_n; i += stride) down_dst[i] = __ldcv(down_src + i);
}

// avirb200_selftest_lin2srgb: every float bit pattern, eight consecutive patterns per thread and step
__global__ void __launch_bounds__(256) lin2srgb_selftest_kernel(unsigned long long* out) {
    unsigned long long checked = 0, bad = 0;
    const unsigned long long nthreads = (unsigned long long)gridDim.x * blockDim.x;
    for (unsigned long long base = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) * 8; base < (1ull << 32);
         base += nthreads * 8) {
        float v[8], ref[8];
        bool ok = true;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            v[i] = __uint_as_float((unsigned)(base + i));
            ok = ok && avb::lin2srgb_batch_ok(v[i]);
        }
        if (!ok) { // (the product takes the one-sample path for such a batch; compare the patterns it accepts singly)
#pragma unroll 1
            for (int i = 0; i < 8; ++i) {
                if (!avb::lin2srgb_batch_ok(v[i])) continue;
                float one[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) one[k] = v[i];
                avb::lin2srgb_batch<8>(one);
                const float r = avb::lin2srgb(v[i]);
                ++checked;
                if (__float_as_uint(r) != __float_as_uint(one[3])) ++bad;
            }
            continue;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) ref[i] = avb::lin2srgb(v[i]);
        avb::lin2srgb_batch<8>(v);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            ++checked;
            if (__float_as_uint(ref[i]) != __float_as_uint(v[i])) ++bad;
        }
    }
    atomicAdd(out, checked);
    atomicAdd(out + 1, bad);
}

void halo_free(Halo* h) {
    if (h == nullptr) return;
    if (h->box_up) cudaIpcCloseMemHandle(h->box_up - h->off_up);
    if (h->box_down) cudaIpcCloseMemHandle(h->box_down - h->off_down);
    // The mailbox itself is NOT freed: a neighbour process may still have it mapped (plans are
    // destroyed without a collective), and freeing exported memory before every importer has closed
    // it is undefined behaviour (CUDA IPC).  A few MB per sharded plan stay allocated until the
    // process ends.
    cudaFreeHost(h->h_seq);
    delete h;
}

// Collective over `comm` (every rank of the sharded call makes it): builds and maps the mailboxes.
// Leaves h->usable false (on EVERY rank) when any rank could not: the NCCL schedule runs then.
int halo_setup(avirb200_plan* pl, void* comm, int rank, int nranks, cudaStream_t st) {
    Nccl* nc = nccl();
    if (!nc) return fail(AVIRB200_ERR_NCCL, "libnccl.so.2 not loadable");
    halo_free(pl->halo);
    Halo* h = pl->halo = new Halo();
    h->comm = comm; h->rank = rank; h->nranks = nranks;
    auto layout = [&](int q, MailboxLayout& l) -> int {
        avirb200_shard_info si;
        const int r = shard_compute(pl, q, nranks, &si);
        if (r == 0) l = MailboxLayout(pl, si);
        return r;
    };
    int r = layout(rank, h->mine);
    if (r == 0 && rank > 0) r = layout(rank - 1, h->above);
    if (r == 0 && rank + 1 < nranks) r = layout(rank + 1, h->below);
    if (r != 0) return r;
    bool ok = nc->AllGather != nullptr;
    cudaIpcMemHandle_t mine;
    std::memset(&mine, 0, sizeof mine);
    // its own allocation (the driver carves small requests out of shared blocks, and an IPC handle
    // names the whole block): at least 2 MiB, in multiples of 2 MiB
    const size_t box_bytes = align_up(h->mine.bytes(2), 2u << 20);
    if (ok) ok = cudaMalloc(&h->box, box_bytes) == cudaSuccess;
    if (ok) ok = cudaMemset(h->box, 0, MailboxLayout::kHeader) == cudaSuccess;
    if (ok) ok = cudaHostAlloc(&h->h_seq, 64 * sizeof(unsigned), cudaHostAllocPortable) == cudaSuccess;
    if (ok) ok = cudaIpcGetMemHandle(&mine, h->box) == cudaSuccess;
    // (an IPC handle names the allocation the pointer lies in; importers add the pointer's offset in it)
    unsigned long long box_off = 0;
    if (ok) {
        typedef int (*RangeFn)(unsigned long long*, size_t*, unsigned long long);
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        unsigned long long base = 0;
        size_t len = 0;
        if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &f, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess && f != nullptr &&
            reinterpret_cast<RangeFn>(f)(&base, &len, (unsigned long long)(uintptr_t)h->box) == 0)
            box_off = (unsigned long long)(uintptr_t)h->box - base;
        else
            cudaGetLastError();
    }
    // all-gather (handle, ok, offset) records
    const size_t rec = sizeof(cudaIpcMemHandle_t) + 16;
    std::vector<char> hostrec((size_t)nranks * rec, 0);
    char* drec = nullptr;
    if (cudaMalloc(&drec, (size_t)nranks * rec) != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_ALLOC, "halo setup"); }
    std::memcpy(&hostrec[(size_t)rank * rec], &mine, sizeof mine);
    hostrec[(size_t)rank * rec + sizeof mine] = ok ? 1 : 0;
    std::memcpy(&hostrec[(size_t)rank * rec + sizeof mine + 8], &box_off, 8);
    cudaMemcpyAsync(drec + (size_t)rank * rec, &hostrec[(size_t)rank * rec], rec, cudaMemcpyHostToDevice, st);
    int nr = nc->AllGather ? nc->AllGather(drec + (size_t)rank * rec, drec, rec, /*ncclChar*/ 0, comm, st) : 1;
    cudaError_t ce = cudaMemcpyAsync(hostrec.data(), drec, (size_t)nranks * rec, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    cudaFree(drec);
    if (nr != 0 || ce != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_NCCL, "halo setup: handle exchange failed"); }
    bool all_ok = true;
    for (int q = 0; q < nranks; ++q) all_ok = all_ok && hostrec[(size_t)q * rec + sizeof mine] == 1;
    // second round: can every rank map its neighbours?
    bool mapped = all_ok;
    if (all_ok && rank > 0) {
        cudaIpcMemHandle_t hh;
        std::memcpy(&hh, &hostrec[(size_t)(rank - 1) * rec], sizeof hh);
        mapped = mapped && cudaIpcOpenMemHandle((void**)&h->box_up, hh, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
        unsigned long long off = 0;
        std::memcpy(&off, &hostrec[(size_t)(rank - 1) * rec + sizeof hh + 8], 8);
        if (mapped) h->box_up += off;
        h->off_up = off;
    }
    if (all_ok && rank + 1 < nranks) {
        cudaIpcMemHandle_t hh;
        std::memcpy(&hh, &hostrec[(size_t)(rank + 1) * rec], sizeof hh);
        mapped = mapped && cudaIpcOpenMemHandle((void**)&h->box_down, hh, cudaIpcMemLazyEnablePeerAccess) == cudaSuccess;
        unsigned long long off = 0;
        std::memcpy(&off, &hostrec[(size_t)(rank + 1) * rec + sizeof hh + 8], 8);
        if (mapped) h->box_down += off;
        h->off_down = off;
    }
    cudaGetLastError();
    std::vector<char> flags((size_t)nranks, 0);
    char* dflag = nullptr;
    if (cudaMalloc(&dflag, (size_t)nranks) != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_ALLOC, "halo setup"); }
    flags[rank] = mapped ? 1 : 0;
    cudaMemcpyAsync(dflag + rank, &flags[rank], 1, cudaMemcpyHostToDevice, st);
    nr = nc->AllGather(dflag + rank, dflag, 1, 0, comm, st);
    ce = cudaMemcpyAsync(flags.data(), dflag, (size_t)nranks, cudaMemcpyDeviceToHost, st);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
    cudaFree(dflag);
    if (nr != 0 || ce != cudaSuccess) { cudaGetLastError(); return fail(AVIRB200_ERR_NCCL, "halo setup: status exchange failed"); }
    bool every = true;
    for (int q = 0; q < nranks; ++q) every = every && flags[q] == 1;
    h->usable = every;
    return 0;
}

// Sharded calls: after the row pass (stream st) the band's boundary rows go to the neighbours' mailboxes on
// the exchange stream (copy engines), each followed by the call's sequence number (at hs).
int sharded_push(avirb200_plan* pl, cudaStream_t st, const float* own, const avs::StreamLink& l, const unsigned* hs) {
    const size_t rowf = mid_pitch(pl);
    const int top_rows = avs::stream_rows_up(l), bot_rows = avs::stream_rows_down(l);
    if (pl->stream_x == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream_x, cudaStreamNonBlocking));
    if (pl->ev_x0 == nullptr) CUDA_TRY(cudaEventCreateWithFlags(&pl->ev_x0, cudaEventDisableTiming));
    if (pl->ev_x1 == nullptr) CUDA_TRY(cudaEventCreateWithFlags(&pl->ev_x1, cudaEventDisableTiming));
    CUDA_TRY(cudaEventRecord(pl->ev_x0, st));
    CUDA_TRY(cudaStreamWaitEvent(pl->stream_x, pl->ev_x0, 0));
    if (top_rows > 0) {
        CUDA_TRY(cudaMemcpyAsync(l.above.from_dn, own, (size_t)top_rows * rowf * 4, cudaMemcpyDefault, pl->stream_x));
        CUDA_TRY(cudaMemcpyAsync(&l.above.flags[1], hs, 4, cudaMemcpyDefault, pl->stream_x));
    }
    if (bot_rows > 0) {
        CUDA_TRY(cudaMemcpyAsync(l.below.from_up, own + (size_t)(l.me->src_rows - bot_rows) * rowf,
                                 (size_t)bot_rows * rowf * 4, cudaMemcpyDefault, pl->stream_x));
        CUDA_TRY(cudaMemcpyAsync(&l.below.flags[0], hs, 4, cudaMemcpyDefault, pl->stream_x));
    }
    CUDA_TRY(cudaEventRecord(pl->ev_x1, pl->stream_x));
    return 0;
}

bool plan_has_f64(const avirb200_plan* pl) { // plans that only run as a whole image through resize_device / _host
    return pl->io_in_type == AVIRB200_F64 || pl->io_out_type == AVIRB200_F64 || pl->errd;
}

} // namespace

extern "C" {

int avirb200_plan_set_option(avirb200_plan* pl, int option, int value) {
    if (pl == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    switch (option) {
    case AVIRB200_OPT_KERNEL_FAMILY: pl->opt_family = (value == 1 || value == 2) ? value : 0; return 0;
    case AVIRB200_OPT_STREAM_VARIANT_H: pl->opt_var_h = (value >= 0 && value < 3) ? value : -1; return 0;
    case AVIRB200_OPT_STREAM_VARIANT_V: pl->opt_var_v = (value >= 0 && value < 3) ? value : -1; return 0;
    case AVIRB200_OPT_HOST_BANDS: pl->opt_host_bands = value >= 1 ? value : -1; return 0;
    case AVIRB200_OPT_OVERLAP_HALO: pl->opt_overlap = (value >= 0 && value <= 3) ? value : 3; return 0;
    case AVIRB200_OPT_ALL_STREAM_CHAINS: {
        const int on = value > 0 ? (value == 2 ? 2 : 1) : 0;
        if (on != pl->opt_all_chains) { // re-decide which passes run on the streaming kernel (host arithmetic only)
            pl->opt_all_chains = on;
            pl->stream_h.chain = pl->stream_v.chain = 0;
            const avirb200_plan_desc& d = pl->desc;
            const int ch = pl->pad4 ? 4 : d.channels;
            if (avs::stream_row_source_ok(d))
                avs::stream_plan_axis(pl->h.desc, d.sum_mode, ch, pl->stream_h, on, false);
            avs::stream_plan_axis(pl->v.desc, d.sum_mode, ch, pl->stream_v, on, true);
        }
        return 0;
    }
    default: return fail(AVIRB200_ERR_BAD_ARG, "unknown option");
    }
}

int avirb200_plan_kernel_paths(const avirb200_plan* pl) {
    if (pl == nullptr) return 0;
    return (pl->stream_h.chain != 0 ? 1 : 0) | (pl->stream_v.chain != 0 ? 2 : 0) |
           (pl->fast.h_ok ? 4 : 0) | (pl->fast.v_ok ? 8 : 0);
}

int avirb200_shard_query_desc(const avirb200_plan_desc* desc, int rank, int nranks,
                              avirb200_shard_info* info) {
    if (desc == nullptr || info == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (desc->v.nsteps < 1 || desc->v.nsteps > AVIRB200_MAX_STEPS)
        return fail(AVIRB200_ERR_BAD_ARG, "axis: nsteps out of range");
    return shard_compute_axis(host_axis_view(desc->v), rank, nranks, info);
}

int avirb200_selftest_lin2srgb(unsigned long long* checked, unsigned long long* mismatches) {
    if (checked == nullptr || mismatches == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    (void)cudaGetLastError();
    unsigned long long* d = nullptr;
    CUDA_TRY(cudaMalloc(&d, 2 * sizeof(unsigned long long)));
    cudaError_t e = cudaMemset(d, 0, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) {
        lin2srgb_selftest_kernel<<<132 * 8, 256>>>(d);
        e = cudaGetLastError();
    }
    unsigned long long h[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpy(h, d, sizeof h, cudaMemcpyDeviceToHost);
    cudaFree(d);
    if (e != cudaSuccess) return fail(AVIRB200_ERR_CUDA, cudaGetErrorString(e));
    *checked = h[0];
    *mismatches = h[1];
    return 0;
}

const char* avirb200_status_string(int s) {
    switch (s) {
    case AVIRB200_OK: return "ok";
    case AVIRB200_ERR_BAD_ARG: return "bad argument";
    case AVIRB200_ERR_CUDA: return "CUDA error";
    case AVIRB200_ERR_NCCL: return "NCCL error";
    case AVIRB200_ERR_UNSUPPORTED: return "unsupported configuration";
    case AVIRB200_ERR_NO_DEVICE: return "no usable CUDA device";
    case AVIRB200_ERR_ALLOC: return "out of memory";
    default: return "unknown status";
    }
}

const char* avirb200_last_error(void) { return g_err.c_str(); }

int avirb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int avirb200_plan_create(const avirb200_plan_desc* desc, avirb200_plan** out) {
    if (desc == nullptr || out == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    *out = nullptr;
    if (desc->channels < 1 || desc->channels > 4 || desc->src_w < 1 || desc->src_h < 1 ||
        desc->dst_w < 1 || desc->dst_h < 1)
        return fail(AVIRB200_ERR_BAD_ARG, "bad image geometry");
    if (desc->in_type < 0 || desc->in_type > 3 || desc->out_type < 0 || desc->out_type > 3)
        return fail(AVIRB200_ERR_BAD_ARG, "bad element type");
    if (desc->h.src_len != desc->src_w || desc->h.dst_len != desc->dst_w ||
        desc->v.src_len != desc->src_h || desc->v.dst_len != desc->dst_h)
        return fail(AVIRB200_ERR_BAD_ARG, "axis lengths do not match the image");
    int ndev = 0;
    {
        cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || ndev == 0)
            return fail(AVIRB200_ERR_NO_DEVICE,
                        std::string("no CUDA device: ") + cudaGetErrorString(e));
    }
    std::unique_ptr<avirb200_plan> pl(new (std::nothrow) avirb200_plan());
    if (!pl) return fail(AVIRB200_ERR_ALLOC, "host allocation failed");
    pl->desc = *desc;
    pl->io_in_type = desc->in_type;
    pl->io_out_type = desc->out_type;
    if (desc->in_type == AVIRB200_F64) pl->desc.in_type = AVIRB200_F32;   // cast on the device first
    if (desc->out_type == AVIRB200_F64) pl->desc.out_type = AVIRB200_F32; // widened on the device last
    if (desc->dither == 1 && (desc->out_type == AVIRB200_U8 || desc->out_type == AVIRB200_U16)) {
        // the column pass delivers the gamma-corrected float rows; errd_kernel rounds them in row order
        pl->errd = true;
        pl->desc.out_type = AVIRB200_F32;
        // errd_kernel's blocks (one warp per 32 rows) wait for their predecessor: keep all of them
        // resident at once (132 SMs x 32 blocks on an H100) instead of relying on in-order block dispatch
        // (32 one-warp blocks per SM; the SM count of the current device, where the plan will live)
        int cur = 0, sms = 0;
        if (cudaGetDevice(&cur) != cudaSuccess ||
            cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cur) != cudaSuccess || sms < 1)
            sms = 1;
        if ((desc->dst_h + 31) / 32 > sms * 32)
            return fail(AVIRB200_ERR_UNSUPPORTED, "error diffusion: more destination rows than the device "
                                                   "keeps resident as one-warp blocks (32 rows each)");
    }
    int r = copy_axis_host(pl->h, desc->h);
    if (r != 0) return r;
    r = copy_axis_host(pl->v, desc->v);
    if (r != 0) return r;
    CUDA_TRY(cudaGetDevice(&pl->device));

    const size_t bytes = axis_arena_bytes(pl->h) + axis_arena_bytes(pl->v) + 1024 + 256;
    CUDA_TRY(cudaMalloc(&pl->arena, bytes));
    std::vector<char> img(bytes, 0);
    size_t off = 0;
    {
        float lut[256];
        make_srgb_lut(lut);
        std::memcpy(img.data(), lut, sizeof lut);
        pl->d_lut = reinterpret_cast<float*>(pl->arena);
        off = 1024;
    }
    build_dev_axis(pl->h, img, off, static_cast<char*>(pl->arena));
    build_dev_axis(pl->v, img, off, static_cast<char*>(pl->arena));
    CUDA_TRY(cudaMemcpy(pl->arena, img.data(), bytes, cudaMemcpyHostToDevice));

    pl->cfg_h = choose_generic_config(pl->h.hostdev, desc->channels, 0, desc->dst_w);
    pl->cfg_v = choose_generic_config(pl->v.hostdev, desc->channels, 0, desc->dst_h);
    // (pl->desc, not *desc: the kernels' element types, see io_in_type / io_out_type)
    // 1..3 channels: can both passes run on the 4-channel kernels (widened copies)?  Not for plans
    // with double buffers or error diffusion (they keep the image's own channel count throughout).
    avirb200_plan_desc d4 = pl->desc;
    const bool try4 = desc->channels < 4 && !(desc->in_type == AVIRB200_F64 || desc->out_type == AVIRB200_F64 || pl->errd);
    if (try4) d4.channels = 4;
    pl->mid_ch = desc->channels;
    fast_plan_init(pl->fast, pl->h.hostdev, pl->v.hostdev, d4);
    // (pl->h.desc / pl->v.desc: the copies whose table pointers stay valid for the plan's life)
    if (avs::stream_row_source_ok(pl->desc))
        avs::stream_plan_axis(pl->h.desc, desc->sum_mode, d4.channels, pl->stream_h, 0, false);
    avs::stream_plan_axis(pl->v.desc, desc->sum_mode, d4.channels, pl->stream_v, 0, true);
    if (try4) {
        const bool h4 = pl->stream_h.chain != 0 || pl->fast.h_ok, v4 = pl->stream_v.chain != 0 || pl->fast.v_ok;
        if (h4 && v4) {
            pl->pad4 = true;
            pl->mid_ch = 4;
        } else { // the image's own channel count on the generic kernel
            pl->stream_h.chain = pl->stream_v.chain = 0;
            pl->fast.h_ok = pl->fast.v_ok = false;
        }
    }
    {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, pl->device) == cudaSuccess && n > 0)
            pl->sm_count = n;
    }
    *out = pl.release();
    return 0;
}

void avirb200_plan_destroy(avirb200_plan* pl) {
    if (pl == nullptr) return;
    cudaFree(pl->arena);
    fast_plan_free(pl->fast);
    halo_free(pl->halo);
    if (pl->stream_x) cudaStreamDestroy(pl->stream_x);
    if (pl->ev_x0) cudaEventDestroy(pl->ev_x0);
    if (pl->ev_x1) cudaEventDestroy(pl->ev_x1);
    if (pl->stream) cudaStreamDestroy(pl->stream);
    if (pl->stream_in) cudaStreamDestroy(pl->stream_in);
    if (pl->stream_out) cudaStreamDestroy(pl->stream_out);
    for (cudaEvent_t e : pl->ev_in) cudaEventDestroy(e);
    for (cudaEvent_t e : pl->ev_out) cudaEventDestroy(e);
    for (cudaEvent_t e : pl->ev_d2h) cudaEventDestroy(e);
    for (cudaEvent_t e : pl->ev_slot) cudaEventDestroy(e);
    delete pl;
}

int avirb200_plan_workspace_bytes(const avirb200_plan* pl, size_t* bytes) {
    if (pl == nullptr || bytes == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    *bytes = ws_layout(pl).total;
    return 0;
}

int avirb200_plan_last_launches(const avirb200_plan* pl) { return pl ? pl->last_launches : 0; }

int avirb200_resize_device(const avirb200_plan* pl, const void* d_src, size_t src_pitch, void* d_dst,
                           size_t dst_pitch, void* d_ws, void* stream) {
    if (pl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    if (src_pitch < (size_t)d.src_w * d.channels || dst_pitch < (size_t)d.dst_w * d.channels)
        return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    {
        int cur = -1;
        if (cudaGetDevice(&cur) != cudaSuccess || cur != pl->device)
            return fail(AVIRB200_ERR_BAD_ARG, "the current device is not the plan's device");
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int launches = 0;
    char* wsb = static_cast<char*>(d_ws);
    const WsLayout ws = ws_layout(pl);
    float* in32 = reinterpret_cast<float*>(wsb + ws.in32);
    float* out32 = reinterpret_cast<float*>(wsb + ws.out32);
    const void* ksrc = d_src;
    size_t ksrc_pitch = src_pitch;
    void* kdst = d_dst;
    size_t kdst_pitch = dst_pitch;
    if (pl->io_in_type == AVIRB200_F64) {
        const int re = d.src_w * d.channels;
        const long long n = (long long)re * d.src_h;
        narrow_f64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(static_cast<const double*>(d_src),
                                                                       (long long)src_pitch, in32, re, d.src_h);
        ++launches;
        ksrc = in32;
        ksrc_pitch = (size_t)re;
    }
    if (pl->io_out_type == AVIRB200_F64 || pl->errd) {
        kdst = out32;
        kdst_pitch = (size_t)d.dst_w * d.channels;
    }
    int r = run_row_pass(pl, ksrc, ksrc_pitch, static_cast<float*>(d_ws), d.src_h, st, &launches, wsb + ws.src4);
    if (r != 0) return r;
    r = run_col_pass(pl, static_cast<const float*>(d_ws), 0, kdst, kdst_pitch, 0, d.dst_h, st,
                     &launches, wsb + ws.dst4);
    if (r == 0 && pl->io_out_type == AVIRB200_F64) {
        const int re = d.dst_w * d.channels;
        const long long n = (long long)re * d.dst_h;
        widen_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out32, static_cast<double*>(d_dst),
                                                                      (long long)dst_pitch, re, d.dst_h);
        ++launches;
        CUDA_TRY(cudaGetLastError());
    }
    if (r == 0 && pl->errd) {
        ErrdParams ep;
        ep.src = out32;
        ep.dst = d_dst;
        ep.dst_pitch = (long long)dst_pitch;
        ep.W = d.dst_w; ep.H = d.dst_h;
        ep.dst_type = pl->io_out_type;
        ep.round_mode = d.round_mode;
        ep.planar = (d.sum_mode == AVIRB200_SUM_DIL8) ? 1 : 0;
        ep.tr_mul = d.tr_mul; ep.tr_mul_inv = d.tr_mul_inv; ep.pk_out = d.pk_out;
        ep.boundary = reinterpret_cast<float*>(wsb + ws.errd_bnd);
        ep.progress = reinterpret_cast<int*>(wsb + ws.errd_prog);
        CUDA_TRY(cudaMemsetAsync(ep.progress, 0, (size_t)errd_groups(pl) * 4, st));
        switch (d.channels) {
        case 1: errd_kernel<1><<<errd_groups(pl), 32, 0, st>>>(ep); break;
        case 2: errd_kernel<2><<<errd_groups(pl), 32, 0, st>>>(ep); break;
        case 3: errd_kernel<3><<<errd_groups(pl), 32, 0, st>>>(ep); break;
        default: errd_kernel<4><<<errd_groups(pl), 32, 0, st>>>(ep); break;
        }
        ++launches;
        CUDA_TRY(cudaGetLastError());
    }
    pl->last_launches = launches;
    return r;
}

int avirb200_row_pass_device(const avirb200_plan* pl, const void* d_src, size_t src_pitch,
                             void* d_ws, void* stream) {
    if (pl == nullptr || d_src == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (plan_has_f64(pl)) return fail(AVIRB200_ERR_UNSUPPORTED, "per-pass entry points: no double buffers, no error diffusion");
    int launches = 0;
    return run_row_pass(pl, d_src, src_pitch, static_cast<float*>(d_ws), pl->desc.src_h,
                        static_cast<cudaStream_t>(stream), &launches, static_cast<char*>(d_ws) + ws_layout(pl).src4);
}

int avirb200_col_pass_device(const avirb200_plan* pl, const void* d_ws, void* d_dst,
                             size_t dst_pitch, void* stream) {
    if (pl == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (plan_has_f64(pl)) return fail(AVIRB200_ERR_UNSUPPORTED, "per-pass entry points: no double buffers, no error diffusion");
    int launches = 0;
    return run_col_pass(pl, static_cast<const float*>(d_ws), 0, d_dst, dst_pitch, 0, pl->desc.dst_h,
                        static_cast<cudaStream_t>(stream), &launches,
                        static_cast<char*>(const_cast<void*>(d_ws)) + ws_layout(pl).dst4);
}

int avirb200_resize_device_batch(const avirb200_plan* pl, int n, const void* const* d_srcs, size_t src_pitch,
                                 void* const* d_dsts, size_t dst_pitch, void* d_ws, void* stream) {
    if (pl == nullptr || d_srcs == nullptr || d_dsts == nullptr || d_ws == nullptr || n < 0)
        return fail(AVIRB200_ERR_BAD_ARG, "bad argument");
    int total = 0;
    for (int i = 0; i < n; ++i) {
        // frames share the workspace: the stream keeps frame i's column pass ahead of frame i+1's row pass
        const int r = avirb200_resize_device(pl, d_srcs[i], src_pitch, d_dsts[i], dst_pitch, d_ws, stream);
        if (r != 0) return r;
        total += pl->last_launches;
    }
    pl->last_launches = total;
    return 0;
}

int avirb200_resize_host(avirb200_plan* pl, const void* h_src, size_t src_pitch, void* h_dst,
                         size_t dst_pitch) {
    if (pl == nullptr || h_src == nullptr || h_dst == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    std::lock_guard<std::mutex> lk(pl->mx);
    // the call runs on the plan's device; the caller's current device is restored on every exit
    struct DeviceGuard {
        int prev = -1;
        ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
    } guard;
    {
        int cur = -1;
        CUDA_TRY(cudaGetDevice(&cur));
        if (cur != pl->device) {
            CUDA_TRY(cudaSetDevice(pl->device));
            guard.prev = cur;
        }
    }
    std::lock_guard<std::mutex> sl(staging_of(pl->device).mx);
    const size_t in_row = (size_t)d.src_w * d.channels * elem_size(pl->io_in_type);
    const size_t out_row = (size_t)d.dst_w * d.channels * elem_size(pl->io_out_type);
    const size_t in_bytes = in_row * d.src_h, out_bytes = out_row * d.dst_h;
    size_t ws = 0;
    avirb200_plan_workspace_bytes(pl, &ws);
    if (pl->stream == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream, cudaStreamNonBlocking));
    {
        const int r0 = plan_staging(pl, in_bytes, out_bytes, ws);
        if (r0 != 0) return r0;
    }
    const size_t in_el = elem_size(pl->io_in_type), out_el = elem_size(pl->io_out_type);
    // Pipelined form for large images: the image is cut into row bands (the multi-GPU band
    // arithmetic, one shared intermediate buffer instead of a halo exchange).  Band b's rows
    // travel host->device on the copy-in stream while the kernels of band b-1 run on the
    // compute stream and band b-2's destination rows travel back on the copy-out stream: the
    // call takes about as long as the larger of the two PCIe directions instead of their sum.
    // The arithmetic does not depend on the banding (tests: 8-band schedule == unsharded bits).
    int nb = (int)(in_bytes >> 25); // bands of >= 32 MiB of source
    if (nb > 16) nb = 16;
    if (pl->opt_host_bands >= 1) nb = pl->opt_host_bands; // test / tuning option
    {   // an aliased or overlapping destination (upstream allows NewBuf == SrcBuf) must not be
        // written before the whole source has been read
        const char* s0 = static_cast<const char*>(h_src);
        const char* d0 = static_cast<const char*>(h_dst);
        const char* s1 = s0 + ((size_t)(d.src_h - 1) * src_pitch + (size_t)d.src_w * d.channels) * in_el;
        const char* d1 = d0 + ((size_t)(d.dst_h - 1) * dst_pitch + (size_t)d.dst_w * d.channels) * out_el;
        if (s0 < d1 && d0 < s1) nb = 1;
    }
    if (plan_has_f64(pl)) nb = 1; // the casts / the row-recursive ditherer run over the whole image
    std::vector<avirb200_shard_info> si;
    while (nb >= 2) { // fewer bands until every band's column pass needs only its neighbours' rows
        si.assign(nb, avirb200_shard_info());
        bool ok = true;
        for (int b = 0; b < nb && ok; ++b) ok = (shard_compute(pl, b, nb, &si[b]) == 0);
        if (ok) break;
        nb /= 2;
    }
    if (nb >= 2) {
        if (pl->stream_in == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream_in, cudaStreamNonBlocking));
        if (pl->stream_out == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream_out, cudaStreamNonBlocking));
        while ((int)pl->ev_in.size() < nb) {
            cudaEvent_t e0, e1;
            CUDA_TRY(cudaEventCreateWithFlags(&e0, cudaEventDisableTiming));
            pl->ev_in.push_back(e0);
            CUDA_TRY(cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
            pl->ev_out.push_back(e1);
        }
        const size_t rowf = mid_pitch(pl);
        const size_t dsrc_pitch = (size_t)d.src_w * d.channels, ddst_pitch = (size_t)d.dst_w * d.channels;
        char* src4 = static_cast<char*>(pl->d_ws) + ws_layout(pl).src4;
        char* dst4 = static_cast<char*>(pl->d_ws) + ws_layout(pl).dst4;
        const size_t src4_row = (size_t)d.src_w * 4 * in_el, dst4_row = (size_t)d.dst_w * 4 * out_el;
        int launches = 0;
        // Pageable (malloc) caller buffers: a copy call straight from / to them returns only when
        // its data has moved (the driver bounces it through its own staging, one thread), which
        // serialises the pipeline.  Such buffers go through the library's page-locked bounce
        // buffers instead, filled / drained by a few host threads: source bands through a ring
        // (a slot is reused once its host->device copy has finished), the destination through a
        // whole-image buffer drained band by band by a helper thread.
        constexpr int kInSlots = 3;
        const bool stage_in = is_pageable(h_src), stage_out = is_pageable(h_dst);
        Staging& sg = staging_of(pl->device);
        size_t slot_bytes = 0;
        for (int b = 0; b < nb; ++b) slot_bytes = std::max(slot_bytes, align_up((size_t)si[b].src_rows * in_row, 4096));
        if (stage_in) { const int r0 = grow_host(&sg.h_in, &sg.h_in_b, slot_bytes * kInSlots); if (r0 != 0) return r0; }
        if (stage_out) { const int r0 = grow_host(&sg.h_out, &sg.h_out_b, out_bytes); if (r0 != 0) return r0; }
        while ((int)pl->ev_slot.size() < kInSlots || (int)pl->ev_d2h.size() < nb) {
            cudaEvent_t e0;
            CUDA_TRY(cudaEventCreateWithFlags(&e0, cudaEventDisableTiming));
            if ((int)pl->ev_slot.size() < kInSlots) pl->ev_slot.push_back(e0); else pl->ev_d2h.push_back(e0);
        }
        // drains destination bands from the bounce buffer into the caller's memory as their copies land
        std::atomic<int> d2h_issued(0), drain_stop(0);
        struct Joiner {
            std::thread t; std::atomic<int>* stop;
            ~Joiner() { if (t.joinable()) { stop->store(1); t.join(); } }
        } drainer{std::thread(), &drain_stop};
        if (stage_out) {
            const int dev = pl->device;
            drainer.t = std::thread([&, dev] {
                cudaSetDevice(dev);
                for (int b = 0; b < nb; ++b) {
                    while (d2h_issued.load() <= b) {
                        if (drain_stop.load()) return;
                        std::this_thread::yield();
                    }
                    if (cudaEventSynchronize(pl->ev_d2h[b]) != cudaSuccess) return;
                    CopyPool::get().copy2d(static_cast<char*>(h_dst) + (size_t)si[b].dst_row0 * dst_pitch * out_el,
                                           dst_pitch * out_el, sg.h_out + (size_t)si[b].dst_row0 * out_row, out_row,
                                           out_row, si[b].dst_rows);
                }
            });
        }
        auto copy_in = [&](int b) -> int {
            if (stage_in) {
                const int slot = b % kInSlots;
                if (b >= kInSlots) CUDA_TRY(cudaEventSynchronize(pl->ev_slot[slot])); // its previous copy has left the slot
                char* hs = sg.h_in + (size_t)slot * slot_bytes;
                CopyPool::get().copy2d(hs, in_row, static_cast<const char*>(h_src) + (size_t)si[b].src_row0 * src_pitch * in_el,
                                       src_pitch * in_el, in_row, si[b].src_rows);
                CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(pl->d_src) + (size_t)si[b].src_row0 * in_row, hs,
                                         (size_t)si[b].src_rows * in_row, cudaMemcpyHostToDevice, pl->stream_in));
                CUDA_TRY(cudaEventRecord(pl->ev_slot[slot], pl->stream_in));
                CUDA_TRY(cudaEventRecord(pl->ev_in[b], pl->stream_in));
                return 0;
            }
            CUDA_TRY(cudaMemcpy2DAsync(static_cast<char*>(pl->d_src) + (size_t)si[b].src_row0 * in_row, in_row,
                                       static_cast<const char*>(h_src) + (size_t)si[b].src_row0 * src_pitch * in_el,
                                       src_pitch * in_el, in_row, si[b].src_rows, cudaMemcpyHostToDevice,
                                       pl->stream_in));
            CUDA_TRY(cudaEventRecord(pl->ev_in[b], pl->stream_in));
            return 0;
        };
        { const int r0 = copy_in(0); if (r0 != 0) return r0; }
        auto col_band = [&](int b) -> int {
            char* dd = static_cast<char*>(pl->d_dst) + (size_t)si[b].dst_row0 * out_row;
            int r = run_col_pass(pl, static_cast<const float*>(pl->d_ws), 0, dd, ddst_pitch, si[b].dst_row0,
                                 si[b].dst_row0 + si[b].dst_rows, pl->stream, &launches,
                                 dst4 + (size_t)si[b].dst_row0 * dst4_row);
            if (r != 0) return r;
            CUDA_TRY(cudaEventRecord(pl->ev_out[b], pl->stream));
            CUDA_TRY(cudaStreamWaitEvent(pl->stream_out, pl->ev_out[b], 0));
            if (stage_out) {
                CUDA_TRY(cudaMemcpyAsync(sg.h_out + (size_t)si[b].dst_row0 * out_row, dd, (size_t)si[b].dst_rows * out_row,
                                         cudaMemcpyDeviceToHost, pl->stream_out));
                CUDA_TRY(cudaEventRecord(pl->ev_d2h[b], pl->stream_out));
                d2h_issued.store(b + 1);
                return 0;
            }
            CUDA_TRY(cudaMemcpy2DAsync(static_cast<char*>(h_dst) + (size_t)si[b].dst_row0 * dst_pitch * out_el,
                                       dst_pitch * out_el, dd, out_row, out_row, si[b].dst_rows,
                                       cudaMemcpyDeviceToHost, pl->stream_out));
            return 0;
        };
        for (int b = 0; b < nb; ++b) {
            if (b + 1 < nb) { const int r0 = copy_in(b + 1); if (r0 != 0) return r0; }
            CUDA_TRY(cudaStreamWaitEvent(pl->stream, pl->ev_in[b], 0));
            int r = run_row_pass(pl, static_cast<const char*>(pl->d_src) + (size_t)si[b].src_row0 * in_row,
                                 dsrc_pitch, static_cast<float*>(pl->d_ws) + (size_t)si[b].src_row0 * rowf,
                                 si[b].src_rows, pl->stream, &launches, src4 + (size_t)si[b].src_row0 * src4_row);
            if (r != 0) return r;
            if (b > 0 && (r = col_band(b - 1)) != 0) return r; // needs rows of bands b-2 .. b only
        }
        int r = col_band(nb - 1);
        if (r != 0) return r;
        pl->last_launches = launches;
        CUDA_TRY(cudaStreamSynchronize(pl->stream_out));
        CUDA_TRY(cudaStreamSynchronize(pl->stream));
        if (drainer.t.joinable()) drainer.t.join(); // the last bands reach the caller's memory
        return 0;
    }
    CUDA_TRY(cudaMemcpy2DAsync(pl->d_src, in_row, h_src, src_pitch * in_el, in_row,
                               d.src_h, cudaMemcpyHostToDevice, pl->stream));
    int r = avirb200_resize_device(pl, pl->d_src, (size_t)d.src_w * d.channels, pl->d_dst,
                                   (size_t)d.dst_w * d.channels, pl->d_ws, pl->stream);
    if (r != 0) return r;
    CUDA_TRY(cudaMemcpy2DAsync(h_dst, dst_pitch * out_el, pl->d_dst, out_row,
                               out_row, d.dst_h, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    return 0;
}

// ---- sharded ---------------------------------------------------------------------------------

int avirb200_shard_query(const avirb200_plan* pl, int rank, int nranks, avirb200_shard_info* info) {
    if (pl == nullptr || info == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const int r = shard_compute(pl, rank, nranks, info);
    // (the tile kernel's table of this destination range: built now, not inside the first launch)
    if (r == 0) fast_prepare_range(pl->fast, info->dst_row0, info->dst_row0 + info->dst_rows);
    return r;
}

int avirb200_shard_workspace_bytes(const avirb200_plan* pl, int rank, int nranks, size_t* bytes) {
    if (pl == nullptr || bytes == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_shard_info si;
    int r = shard_compute(pl, rank, nranks, &si);
    if (r != 0) return r;
    fast_prepare_range(pl->fast, si.dst_row0, si.dst_row0 + si.dst_rows);
    *bytes = ws_layout(pl, si).total;
    return 0;
}

int avirb200_comm_unique_id(void* id128) {
    Nccl* nc = nccl();
    if (!nc) return fail(AVIRB200_ERR_NCCL, "libnccl.so.2 not loadable");
    NCCL_TRY(nc->GetUniqueId(id128));
    return 0;
}

int avirb200_comm_create(const void* id128, int rank, int nranks, void** comm_out) {
    Nccl* nc = nccl();
    if (!nc) return fail(AVIRB200_ERR_NCCL, "libnccl.so.2 not loadable");
    Id128 id;
    std::memcpy(&id, id128, sizeof id);
    NCCL_TRY(nc->CommInitRank(comm_out, nranks, id, rank));
    return 0;
}

void avirb200_comm_destroy(void* comm) {
    Nccl* nc = nccl();
    if (nc && nc->CommDestroy && comm) nc->CommDestroy(comm);
}

int avirb200_resize_sharded(const avirb200_plan* cpl, void* comm, int rank, int nranks,
                            const void* d_src, size_t src_pitch, void* d_dst, size_t dst_pitch,
                            void* d_ws, void* stream) {
    if (cpl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_plan* pl = const_cast<avirb200_plan*>(cpl); // (exchange state is created on first use)
    if (plan_has_f64(pl)) return fail(AVIRB200_ERR_UNSUPPORTED, "sharded calls: no double buffers, no error diffusion");
    { int cur = -1; if (cudaGetDevice(&cur) != cudaSuccess || cur != pl->device) return fail(AVIRB200_ERR_BAD_ARG, "the current device is not the plan's device"); }
    avirb200_shard_info si;
    int r = shard_compute(pl, rank, nranks, &si);
    if (r != 0) return r;
    const avirb200_plan_desc& d = pl->desc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t rowf = mid_pitch(pl);
    const size_t in_el = elem_size(d.in_type);
    float* mid = static_cast<float*>(d_ws);
    float* own = mid + (size_t)si.halo_up * rowf;
    const WsLayout ws = ws_layout(pl, si);
    char* src4 = static_cast<char*>(d_ws) + ws.src4;
    char* dst4 = static_cast<char*>(d_ws) + ws.dst4;
    const size_t src4_row = (size_t)d.src_w * 4 * in_el;
    int launches = 0;
    if (nranks <= 1) {
        r = run_row_pass(pl, d_src, src_pitch, own, si.src_rows, st, &launches, src4);
        if (r != 0) return r;
        r = run_col_pass(pl, mid, si.need_row0, d_dst, dst_pitch, si.dst_row0, si.dst_row0 + si.dst_rows, st, &launches, dst4,
                         si.need_rows);
        pl->last_launches = launches;
        return r;
    }
    if (comm == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "sharded resize needs a communicator");
    Nccl* nc = nccl();
    if (!nc) return fail(AVIRB200_ERR_NCCL, "libnccl.so.2 not loadable");
    // What the neighbours need from this rank is symmetric information: compute theirs.
    avirb200_shard_info up, down;
    std::memset(&up, 0, sizeof up); std::memset(&down, 0, sizeof down);
    if (rank > 0) { r = shard_compute(pl, rank - 1, nranks, &up); if (r != 0) return r; }
    if (rank + 1 < nranks) { r = shard_compute(pl, rank + 1, nranks, &down); if (r != 0) return r; }
    avs::StreamLink link; // (the mailboxes are filled in below)
    link.me = &si;
    link.up = (rank > 0) ? &up : nullptr;
    link.dn = (rank + 1 < nranks) ? &down : nullptr;
    const int top_rows = avs::stream_rows_up(link), bot_rows = avs::stream_rows_down(link);

    std::lock_guard<std::mutex> lk(pl->mx);
    if (pl->opt_overlap) {
        if (pl->halo == nullptr || pl->halo->comm != comm || pl->halo->rank != rank || pl->halo->nranks != nranks) {
            r = halo_setup(pl, comm, rank, nranks, st); // collective, once per plan
            if (r != 0) return r;
        }
    }
    Halo* h = (pl->opt_overlap && pl->halo && pl->halo->usable) ? pl->halo : nullptr;
    if (h != nullptr) {
        const unsigned seq = ++h->seq;
        const int slot = (int)(seq & 1u);
        unsigned* hs = &h->h_seq[seq & 63u];
        *hs = seq;
        const char* srcb = static_cast<const char*>(d_src);
        auto rows_pass = [&](int row0, int nrows) -> int {
            if (nrows <= 0) return 0;
            return run_row_pass(pl, srcb + (size_t)row0 * src_pitch * in_el, src_pitch, own + (size_t)row0 * rowf,
                                nrows, st, &launches, src4 + (size_t)row0 * src4_row);
        };
        const int need_up = (link.up && si.halo_up > 0) ? 1 : 0;
        const int need_down = (link.dn && si.halo_down > 0) ? 1 : 0;
        link.seq = seq;
        link.mine = h->mine.at(h->box, slot);
        if (link.up) link.above = h->above.at(h->box_up, slot);
        if (link.dn) link.below = h->below.at(h->box_down, slot);
        // AVIRB200_OPT_OVERLAP_HALO = 3, the fused exchange: the row kernel stores the rows the neighbours need
        // into their mailboxes as it produces them (peer stores over NVLink) and raises their flags when the
        // last of them is out; the column kernel reads the neighbours' rows in place from this rank's mailbox,
        // waiting on the flags only in the runs that touch them.  No exchange stream, no copy, no extra launch.
        // Either half falls back on its own (the mailbox protocol is the same): a row pass that is not on the
        // streaming kernel pushes with the copy engines, a column pass that is not pulls into the workspace.
        const bool fused = pl->opt_overlap == 3 && avs::stream_fused_rx_ok(link);
        const bool fused_tx = pl->opt_overlap == 3 && avs::stream_fused_tx_ok(link);
        bool sent = false, pushed = false;
        if (fused_tx && top_rows + bot_rows > 0) {
            if ((r = run_row_pass(pl, d_src, src_pitch, own, si.src_rows, st, &launches, src4, 0, 0, &link, &sent)) != 0) return r;
        } else {
            // 1. the rows the neighbours need (one launch on the streaming kernel: two line segments),
            // 2. their push on the exchange stream, 3. the interior rows
            // (boundary rows first only on request, AVIRB200_OPT_OVERLAP_HALO = 2: the copy-engine push
            // of cfg3's 1.2 MB is short next to the extra launch the split costs)
            const bool split = pl->opt_overlap == 2 && top_rows + bot_rows < si.src_rows;
            if (split && !use_pad4(pl) && row_pass_on_stream(pl, d_src, src_pitch, own)) {
                if (top_rows + bot_rows > 0 &&
                    (r = run_row_pass(pl, d_src, src_pitch, own, si.src_rows, st, &launches, nullptr, top_rows, bot_rows)) != 0)
                    return r;
            } else if (split) {
                if ((r = rows_pass(0, top_rows)) != 0) return r;
                if ((r = rows_pass(si.src_rows - bot_rows, bot_rows)) != 0) return r;
            } else if ((r = rows_pass(0, si.src_rows)) != 0) {
                return r;
            }
            if ((r = sharded_push(pl, st, own, link, hs)) != 0) return r;
            sent = pushed = true;
            if (split && (r = rows_pass(top_rows, si.src_rows - top_rows - bot_rows)) != 0) return r;
        }
        if (!sent && top_rows + bot_rows > 0) { // the fused row pass did not run on the streaming kernel
            if ((r = sharded_push(pl, st, own, link, hs)) != 0) return r;
            pushed = true;
        }
        // 4. the neighbours' rows: in place (fused), or wait for their sequence numbers and move them
        // mailbox -> workspace
        r = 1;
        if (fused && (need_up || need_down)) {
            r = run_col_pass(pl, mid, si.need_row0, d_dst, dst_pitch, si.dst_row0, si.dst_row0 + si.dst_rows, st, &launches,
                             dst4, si.need_rows, &link);
        }
        if (r == 1) {
            if (need_up || need_down) {
                (void)cudaGetLastError();
                halo_pull_kernel<<<64, 256, 0, st>>>(link.mine.flags, seq, need_up, need_down,
                                                     reinterpret_cast<const float4*>(link.mine.from_up), reinterpret_cast<float4*>(mid),
                                                     need_up ? h->mine.up_bytes / 16 : 0,
                                                     reinterpret_cast<const float4*>(link.mine.from_dn),
                                                     reinterpret_cast<float4*>(own + (size_t)si.src_rows * rowf),
                                                     need_down ? h->mine.down_bytes / 16 : 0);
                ++launches;
                CUDA_TRY(cudaGetLastError());
            }
            r = run_col_pass(pl, mid, si.need_row0, d_dst, dst_pitch, si.dst_row0, si.dst_row0 + si.dst_rows, st, &launches,
                             dst4, si.need_rows);
        }
        // the pushes read this call's workspace: the caller's stream does not end before them
        if (pushed) CUDA_TRY(cudaStreamWaitEvent(st, pl->ev_x1, 0));
        pl->last_launches = launches;
        return r;
    }
    // NCCL schedule: whole row pass, send/recv group, column pass, one stream
    r = run_row_pass(pl, d_src, src_pitch, own, si.src_rows, st, &launches, src4);
    if (r != 0) return r;
    NCCL_TRY(nc->GroupStart());
    if (rank > 0) {
        if (top_rows > 0) NCCL_TRY(nc->Send(own, (size_t)top_rows * rowf, 7, rank - 1, comm, st));
        if (si.halo_up > 0) NCCL_TRY(nc->Recv(mid, (size_t)si.halo_up * rowf, 7, rank - 1, comm, st));
    }
    if (rank + 1 < nranks) {
        if (bot_rows > 0)
            NCCL_TRY(nc->Send(own + (size_t)(si.src_rows - bot_rows) * rowf, (size_t)bot_rows * rowf, 7, rank + 1, comm, st));
        if (si.halo_down > 0)
            NCCL_TRY(nc->Recv(own + (size_t)si.src_rows * rowf, (size_t)si.halo_down * rowf, 7, rank + 1, comm, st));
    }
    NCCL_TRY(nc->GroupEnd());
    r = run_col_pass(pl, mid, si.need_row0, d_dst, dst_pitch, si.dst_row0, si.dst_row0 + si.dst_rows, st, &launches, dst4,
                     si.need_rows);
    pl->last_launches = launches;
    return r;
}

int avirb200_resize_sharded_host(avirb200_plan* pl, void* comm, int rank, int nranks, const void* h_src,
                                 size_t src_pitch, void* h_dst, size_t dst_pitch) {
    if (pl == nullptr || h_src == nullptr || h_dst == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (plan_has_f64(pl)) return fail(AVIRB200_ERR_UNSUPPORTED, "sharded calls: no double buffers, no error diffusion");
    const avirb200_plan_desc& d = pl->desc;
    avirb200_shard_info si;
    int r = shard_compute(pl, rank, nranks, &si);
    if (r != 0) return r;
    size_t ws = 0;
    if ((r = avirb200_shard_workspace_bytes(pl, rank, nranks, &ws)) != 0) return r;
    const size_t in_row = (size_t)d.src_w * d.channels * elem_size(d.in_type);
    const size_t out_row = (size_t)d.dst_w * d.channels * elem_size(d.out_type);
    {
        std::lock_guard<std::mutex> lk(pl->mx);
        int cur = -1;
        if (cudaGetDevice(&cur) != cudaSuccess || cur != pl->device)
            return fail(AVIRB200_ERR_BAD_ARG, "the current device is not the plan's device");
        if (pl->stream == nullptr) CUDA_TRY(cudaStreamCreateWithFlags(&pl->stream, cudaStreamNonBlocking));
    }
    std::lock_guard<std::mutex> sl(staging_of(pl->device).mx);
    r = plan_staging(pl, in_row * si.src_rows, out_row * si.dst_rows, ws);
    if (r != 0) return r;
    CUDA_TRY(cudaMemcpy2DAsync(pl->d_src, in_row, h_src, src_pitch * elem_size(d.in_type), in_row, si.src_rows,
                               cudaMemcpyHostToDevice, pl->stream));
    r = avirb200_resize_sharded(pl, comm, rank, nranks, pl->d_src, (size_t)d.src_w * d.channels, pl->d_dst,
                                (size_t)d.dst_w * d.channels, pl->d_ws, pl->stream);
    if (r != 0) return r;
    CUDA_TRY(cudaMemcpy2DAsync(h_dst, dst_pitch * elem_size(d.out_type), pl->d_dst, out_row, out_row, si.dst_rows,
                               cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    return 0;
}

int avirb200_resize_sharded_local(const avirb200_plan* pl, int nranks, const void* d_src,
                                  size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws,
                                  void* stream) {
    if (pl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (plan_has_f64(pl)) return fail(AVIRB200_ERR_UNSUPPORTED, "sharded calls: no double buffers, no error diffusion");
    const avirb200_plan_desc& d = pl->desc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t rowf = mid_pitch(pl);
    const size_t in_el = elem_size(d.in_type), out_el = elem_size(d.out_type);
    std::vector<avirb200_shard_info> si(nranks);
    std::vector<float*> mid(nranks), own(nranks);
    std::vector<const char*> src(nranks);
    std::vector<char*> dst(nranks), src4(nranks), dst4(nranks);
    char* base = static_cast<char*>(d_ws);
    for (int r = 0; r < nranks; ++r) { // every band's segment: as avirb200_shard_workspace_bytes lays it out
        int e = shard_compute(pl, r, nranks, &si[r]);
        if (e != 0) return e;
        const WsLayout ws = ws_layout(pl, si[r]);
        mid[r] = reinterpret_cast<float*>(base);
        own[r] = mid[r] + (size_t)si[r].halo_up * rowf;
        src4[r] = base + ws.src4;
        dst4[r] = base + ws.dst4;
        base += ws.total;
        src[r] = static_cast<const char*>(d_src) + (size_t)si[r].src_row0 * src_pitch * in_el;
        dst[r] = static_cast<char*>(d_dst) + (size_t)si[r].dst_row0 * dst_pitch * out_el;
    }
    int launches = 0;
    // The fused halo exchange of avirb200_resize_sharded (AVIRB200_OPT_OVERLAP_HALO = 3), with every band's
    // mailbox (one slot) in this device's memory: the same two kernels, parameters and protocol as between
    // ranks.  Only when every band may run both fused halves and both its passes run on the streaming kernel
    // (a widened plan's kernels see its scratch copies).
    const bool p4 = use_pad4(pl);
    std::vector<avs::StreamLink> link(nranks);
    std::vector<MailboxLayout> box(nranks);
    std::vector<size_t> box_off(nranks + 1, 0);
    bool fused = pl->opt_overlap == 3 && nranks > 1;
    for (int r = 0; r < nranks && fused; ++r) {
        link[r].me = &si[r];
        if (r > 0) link[r].up = &si[r - 1];
        if (r + 1 < nranks) link[r].dn = &si[r + 1];
        fused = avs::stream_fused_tx_ok(link[r]) &&
                row_pass_on_stream(pl, p4 ? src4[r] : src[r], p4 ? (size_t)d.src_w * 4 : src_pitch, own[r]) &&
                col_pass_on_stream(pl, p4 ? dst4[r] : dst[r], p4 ? (size_t)d.dst_w * 4 : dst_pitch, mid[r]);
        box[r] = MailboxLayout(pl, si[r]);
        box_off[r + 1] = box_off[r] + box[r].bytes(1);
    }
    if (fused) {
        char* boxes = nullptr;
        CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&boxes), box_off[nranks], st));
        int e = 0;
        for (int r = 0; r < nranks; ++r) {
            link[r].mine = box[r].at(boxes + box_off[r], 0);
            link[r].seq = 1;
            if (e == 0 && cudaMemsetAsync(boxes + box_off[r], 0, MailboxLayout::kHeader, st) != cudaSuccess)
                e = fail(AVIRB200_ERR_CUDA, "sharded_local: mailbox header");
        }
        for (int r = 0; r < nranks; ++r) {
            if (r > 0) link[r].above = link[r - 1].mine;
            if (r + 1 < nranks) link[r].below = link[r + 1].mine;
        }
        for (int r = 0; r < nranks && e == 0; ++r) {
            const bool tx = avs::stream_rows_up(link[r]) + avs::stream_rows_down(link[r]) > 0;
            bool sent = false;
            e = run_row_pass(pl, src[r], src_pitch, own[r], si[r].src_rows, st, &launches, src4[r], 0, 0,
                             tx ? &link[r] : nullptr, &sent);
            if (e == 0 && tx && !sent) e = fail(AVIRB200_ERR_CUDA, "sharded_local: the streaming row pass did not take the band");
        }
        for (int r = 0; r < nranks && e == 0; ++r) {
            e = run_col_pass(pl, mid[r], si[r].need_row0, dst[r], dst_pitch, si[r].dst_row0, si[r].dst_row0 + si[r].dst_rows,
                             st, &launches, dst4[r], si[r].need_rows, &link[r]);
            if (e == 1) e = fail(AVIRB200_ERR_CUDA, "sharded_local: the streaming column pass did not take the band");
        }
        cudaFreeAsync(boxes, st);
        pl->last_launches = launches;
        return e;
    }
    for (int r = 0; r < nranks; ++r) { // every band's row pass
        int e = run_row_pass(pl, src[r], src_pitch, own[r], si[r].src_rows, st, &launches, src4[r]);
        if (e != 0) return e;
    }
    for (int r = 0; r < nranks; ++r) { // the "exchange"
        if (r > 0 && si[r].halo_up > 0) {
            const float* nb = own[r - 1] + (size_t)(si[r - 1].src_rows - si[r].halo_up) * rowf;
            CUDA_TRY(cudaMemcpyAsync(mid[r], nb, (size_t)si[r].halo_up * rowf * 4,
                                     cudaMemcpyDeviceToDevice, st));
        }
        if (r + 1 < nranks && si[r].halo_down > 0) {
            CUDA_TRY(cudaMemcpyAsync(own[r] + (size_t)si[r].src_rows * rowf, own[r + 1],
                                     (size_t)si[r].halo_down * rowf * 4, cudaMemcpyDeviceToDevice, st));
        }
    }
    for (int r = 0; r < nranks; ++r) {
        int e = run_col_pass(pl, mid[r], si[r].need_row0, dst[r], dst_pitch, si[r].dst_row0,
                             si[r].dst_row0 + si[r].dst_rows, st, &launches, dst4[r], si[r].need_rows);
        if (e != 0) return e;
    }
    pl->last_launches = launches;
    return 0;
}

} // extern "C"
