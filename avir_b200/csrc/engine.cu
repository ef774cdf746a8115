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
#include "host_call.h"
#include "host_util.h"
#include "pass_config.h"
#include "pass_request.h"
#include "peer_mailbox.h"
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

struct HostAxis {
    avirb200_axis_desc desc;              // pointers are HOST copies (below)
    std::vector<std::vector<float> > taps, frac, pdc, sdc;
    std::vector<std::vector<int32_t> > src_pos, phase;
    DevAxis dev;                          // device pointers
    DevAxis hostdev;                      // same geometry, host src_pos pointers (range math)
};

} // namespace

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
    // held by host calls (host_call.h) and by sharded calls of more than one rank; host calls run on `stream`
    std::mutex mx;
    cudaStream_t stream = nullptr;
    // pipelined resize_host: copy-in / copy-out streams and per-band events
    cudaStream_t stream_in = nullptr, stream_out = nullptr;
    std::vector<cudaEvent_t> ev_in, ev_out, ev_d2h, ev_slot; // (+ staged copies of pageable buffers)
    // launches of the last call that counted them; calls on one plan from several threads each store their
    // own count (relaxed: the value is some one call's, never a mix)
    mutable std::atomic<int> last_launches{0};
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
    size_t smem_optin = 232448; // of `device`: the most dynamic shared memory one block may opt in to
    PeerExchange x;           // sharded: the halo exchange (opened by the first sharded call of more than one rank)
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

// grid.y: the blocks of lines, at most 65535 (the kernel loops over the rest).
int launch_generic(const PassParams& p, const PassConfig& c, cudaStream_t st) {
    const int line_blocks = (p.n_lines + c.lines_per_block - 1) / c.lines_per_block;
    dim3 grid((p.out1 - p.out0 + c.tile_out - 1) / c.tile_out, imin(line_blocks, 65535));
    if (grid.x == 0 || grid.y == 0) return 0;
    if (p.sum_mode == AVIRB200_SUM_DIL8) {
        CUDA_TRY(raise_smem_limit(reinterpret_cast<const void*>(generic_pass_kernel<AVIRB200_SUM_DIL8>), c.smem));
        generic_pass_kernel<AVIRB200_SUM_DIL8><<<grid, 256, c.smem, st>>>(p);
    } else {
        CUDA_TRY(raise_smem_limit(reinterpret_cast<const void*>(generic_pass_kernel<AVIRB200_SUM_INL>), c.smem));
        generic_pass_kernel<AVIRB200_SUM_INL><<<grid, 256, c.smem, st>>>(p);
    }
    CUDA_TRY(cudaGetLastError());
    return 0;
}

int launch_widen(int type, const void* src, size_t src_pitch, void* dst, int w, int rows, int C, cudaStream_t st);
int launch_narrow(int type, const void* src, void* dst, size_t dst_pitch, int w, int rows, int C, cudaStream_t st);

// 1..3-channel plans whose passes run on the 4-channel kernels in this call (avirb200_plan::pad4)
bool use_pad4(const avirb200_plan* pl) { return pl->pad4 && pl->opt_family != 1; }

// Floats between consecutive intermediate rows, for every kernel family and every band / halo offset
// (cols: the intermediate columns a window's passes run over; < 0: the whole destination width).
size_t mid_pitch(const avirb200_plan* pl, int cols = -1) {
    return (size_t)(cols >= 0 ? cols : pl->desc.dst_w) * pl->mid_ch;
}

enum PassFamily { kFamilyStream, kFamilyTile, kFamilyGeneric };

struct PassRoute {
    PassFamily family;
    PassRequest k;      // the request as the kernels see it: a widened plan's scratch copies
    FastFootprint fpnt; // kFamilyTile: the footprint of the request's range
    const int* tiles = nullptr; // kFamilyTile: the range's tile table
};

// The kernel family that runs the pass `req`: the first that applies of the streaming kernel, the tile
// kernel and the generic kernel.  The 4-channel kernels (streaming, tile) move whole pixels: the row pass's
// source pixels and the column pass's channel pairs must be aligned to their size, the intermediate to 16
// bytes.  The tile kernel also needs the table of the request's range, built ahead by plan creation, a window or
// shard query or the banded host call (a launch never builds one: no allocation, no synchronous copy), and the
// footprint of the range's tiles to fit its shared memory.
PassRoute pass_family(const avirb200_plan* pl, const PassRequest& req) {
    PassRoute r;
    r.k = req;
    PassRequest& k = r.k;
    if (use_pad4(pl)) {
        if (k.is_v) {
            k.dst = k.scratch4;
            k.dst_pitch = (size_t)k.lines * 4;
        } else {
            k.src = k.scratch4;
            k.src_pitch = (size_t)(k.src_hi - k.src_lo) * 4;
        }
    }
    const bool aligned = k.is_v ? ((uintptr_t)k.dst % (2 * elem_size(k.dst_type))) == 0 && (k.dst_pitch % 2) == 0 &&
                                      ((uintptr_t)k.src % 16) == 0
                                : ((uintptr_t)k.src % (4 * elem_size(k.src_type))) == 0 && (k.src_pitch % 4) == 0 &&
                                      ((uintptr_t)k.dst % 16) == 0;
    const avs::StreamAxisPlan& sa = k.is_v ? pl->stream_v : pl->stream_h;
    const bool tile_ok = k.is_v ? pl->fast.v_ok : pl->fast.h_ok;
    const FastPass& fp = k.is_v ? pl->fast.v : pl->fast.h;
    if (pl->opt_family == 0 && sa.chain != 0 && aligned) {
        r.family = kFamilyStream;
    } else if (pl->opt_family != 1 && tile_ok && aligned && (r.tiles = fast_tile_table_find(fp, k.out0, k.out1)) != nullptr &&
               (r.fpnt = fast_range_footprint(fp, k.out0, k.out1)).smem <= kFastSmemBudget) {
        r.family = kFamilyTile;
    } else {
        r.family = kFamilyGeneric;
    }
    return r;
}

// The generic kernel's parameters of the pass k (its buffers as the kernel sees them), `channels` wide: the
// plan's cached layout for a whole pass at the image's channel count, else the range's own.
int generic_pass(const avirb200_plan* pl, const PassRequest& k, int channels, cudaStream_t st) {
    const avirb200_plan_desc& d = pl->desc;
    const HostAxis& ax = k.is_v ? pl->v : pl->h;
    const PassConfig c = (channels == d.channels && k.out0 == 0 && k.out1 == ax.desc.dst_len)
                             ? (k.is_v ? pl->cfg_v : pl->cfg_h)
                             : choose_generic_config(ax.hostdev, channels, k.out0, k.out1, pl->smem_optin);
    PassParams p;
    std::memset(&p, 0, sizeof p);
    p.ax = ax.dev;
    p.sum_mode = d.sum_mode;
    p.is_v = k.is_v ? 1 : 0;
    p.channels = channels;
    p.n_lines = k.lines;
    p.lines_per_block = c.lines_per_block;
    p.tile_out = c.tile_out;
    p.out0 = k.out0;
    p.out1 = k.out1;
    p.span_a = c.span_a;
    p.pitch = c.pitch;
    p.src = k.src;
    p.src_pitch = (long long)k.src_pitch;
    p.src_type = k.src_type;
    p.src_row_base = k.src_base;
    p.dst = k.dst;
    p.dst_pitch = (long long)k.dst_pitch;
    p.dst_type = k.dst_type;
    p.dst_row_base = k.dst_base;
    p.px = pixel_stage(d, pl->d_lut);
    return launch_generic(p, c, st);
}

// Runs one pass on the family pass_family() picks.  A widened plan's row pass first widens the source
// into req.scratch4, its column pass writes 4-channel pixels there and narrows them into req.dst; a widened
// pass the 4-channel kernels do not take runs the generic kernel with 4 channels (the pad channel's results
// are dropped).  Line segments and links are the streaming kernel's: the caller asks pass_family() first.
int run_pass(const avirb200_plan* pl, const PassRequest& req, cudaStream_t st, int* launches) {
    if (req.lines <= 0 || req.out1 <= req.out0) return 0;
    // (a non-sticky error another library left in this thread -- NCCL's peer-access probing leaves
    // cudaErrorPeerAccessAlreadyEnabled once the IPC mailboxes have enabled it -- is not this launch's)
    (void)cudaGetLastError();
    const avirb200_plan_desc& d = pl->desc;
    const char* pass = req.is_v ? "column pass" : "row pass";
    const bool p4 = use_pad4(pl);
    if (p4 && req.scratch4 == nullptr) return fail(AVIRB200_ERR_BAD_ARG, std::string(pass) + ": no scratch for the widened pixels");
    const PassRoute r = pass_family(pl, req);
    const PassRequest& k = r.k;
    if ((k.link != nullptr || k.seg_top > 0 || k.seg_bot > 0) && r.family != kFamilyStream)
        return fail(AVIRB200_ERR_BAD_ARG, std::string(pass) + ": line segments and links need the streaming kernel");
    if (p4 && !k.is_v) {
        if (launch_widen(d.in_type, req.src, req.src_pitch, req.scratch4, k.src_hi - k.src_lo, k.lines, d.channels, st) != 0)
            return fail(AVIRB200_ERR_CUDA, "widening the source failed");
        ++*launches;
    }
    int e = 0;
    if (r.family == kFamilyStream) {
        const avs::StreamAxisPlan& sa = k.is_v ? pl->stream_v : pl->stream_h;
        avs::StreamParams sp;
        avs::stream_params(sp, sa, d, k, pl->d_lut);
        if (avs::stream_launch(sa.chain, k.is_v, avs::stream_epilogue_code(d), k.is_v ? pl->opt_var_v : pl->opt_var_h, sp,
                               pl->sm_count, st) != 0)
            e = fail(AVIRB200_ERR_CUDA, std::string("streaming ") + pass + " launch failed");
    } else if (r.family == kFamilyTile) {
        if (fast_pass(k.is_v ? pl->fast.v : pl->fast.h, k, r.fpnt, r.tiles, pixel_stage(d, pl->d_lut), d.sum_mode,
                      pl->sm_count, st) != 0)
            e = fail(AVIRB200_ERR_CUDA, std::string("fast ") + pass + " launch failed");
    } else {
        e = generic_pass(pl, k, p4 ? 4 : d.channels, st);
    }
    if (e != 0) return e;
    ++*launches;
    if (p4 && k.is_v) {
        if (launch_narrow(d.out_type, k.dst, req.dst, req.dst_pitch, k.lines, k.out1 - k.out0, d.channels, st) != 0)
            return fail(AVIRB200_ERR_CUDA, "narrowing the destination failed");
        ++*launches;
    }
    return 0;
}

// The bands of rank `rank` of `nranks`; need_*: the intermediate rows its column pass reads.
int shard_compute_axis(const DevAxis& vaxis, int rank, int nranks, avirb200_shard_info* info) {
    int r = shard_split(vaxis.src_len, vaxis.dst_len, rank, nranks, info);
    if (r != 0) return r;
    const Range need = chain_source_range(vaxis, Range{info->dst_row0, info->dst_row0 + info->dst_rows - 1}, nullptr);
    return shard_halos(need.a, need.b + 1, vaxis.src_len, rank, nranks, info);
}

int shard_compute(const avirb200_plan* pl, int rank, int nranks, avirb200_shard_info* info) {
    return shard_compute_axis(pl->v.hostdev, rank, nranks, info);
}

// A destination window's footprint: the source columns / rows both chains read for it.  errd: the plan
// diffuses the rounding error (a window of it is not a window of the whole image's result).
int window_compute(const DevAxis& h, const DevAxis& v, bool errd, int x0, int y0, int w, int hh,
                   avirb200_window_info* info) {
    if (w < 1 || hh < 1 || x0 < 0 || y0 < 0 || (long long)x0 + w > h.dst_len || (long long)y0 + hh > v.dst_len)
        return fail(AVIRB200_ERR_BAD_ARG, "window empty or outside the destination");
    if (errd) return fail(AVIRB200_ERR_UNSUPPORTED, "windows: error diffusion depends on every pixel before the window");
    const Range cx = chain_source_range(h, Range{x0, x0 + w - 1}, nullptr);
    const Range cy = chain_source_range(v, Range{y0, y0 + hh - 1}, nullptr);
    info->src_x0 = cx.a;
    info->src_w = cx.b - cx.a + 1;
    info->src_y0 = info->mid_row0 = cy.a;
    info->src_h = info->mid_rows = cy.b - cy.a + 1;
    return 0;
}

int window_compute(const avirb200_plan* pl, int x0, int y0, int w, int h, avirb200_window_info* info) {
    const int r = window_compute(pl->h.hostdev, pl->v.hostdev, pl->errd, x0, y0, w, h, info);
    // (the tile kernel's tables of the window's column and row ranges: built now, not inside a launch)
    if (r == 0) {
        fast_prepare_columns(pl->fast, x0, x0 + w);
        fast_prepare_range(pl->fast, y0, y0 + h);
    }
    return r;
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
// A band of a sharded call runs the same kernel over its own rows: its first group takes the D row of
// the band above (carry_in) instead of zeros, and its last row publishes its D row (carry_out) to the
// band below the way lane 31 publishes to the next group.  The result does not depend on the banding.
struct ErrdParams {
    const float* src;     // [H][W*C] gamma-corrected floats (the column pass's output)
    void* dst;
    long long dst_pitch;  // elements
    int W, H, dst_type, round_mode;
    int planar;           // de-interleaved class: channel c+1's pixel 0 also feeds channel c's last D (see below)
    float tr_mul, tr_mul_inv, pk_out;
    float* boundary;      // [groups][W*C]
    int* progress;        // [groups]: pixels of the group's last row whose D values are published
    // carry_in: D of row 0 (null: zeros, the image's first row).  carry_in_prog null: carry_in is complete
    // before the launch; else a progress word (seq << 32 | pixels published), see errd_carry_ready.
    const float* carry_in;
    const unsigned long long* carry_in_prog;
    // carry_out: D of the row below row H-1 (null: no band below).  carry_out_prog null: nobody waits for
    // it (a copy follows the kernel); else seq << 32 | pixels published, after a system-scope fence.
    float* carry_out;
    unsigned long long* carry_out_prog;
    unsigned seq; // the call's sequence number: a progress word names its call, so it is never reset
};

// Whether progress word v (seq << 32 | pixels) shows pixel pix of call seq published.  The sequence halves are
// compared modulo 2^32 (as the halo flags are): a word of an earlier call is older even after seq wraps.
__device__ __forceinline__ bool errd_carry_ready(unsigned long long v, unsigned seq, int pix) {
    const unsigned hi = (unsigned)(v >> 32), lo = (unsigned)v;
    return hi == seq ? lo > (unsigned)pix : (int)(hi - seq) > 0;
}

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
    const bool carry = p.carry_out != nullptr && y == p.H - 1; // the band's last row: publishes to the band below
    int seen = 0; // lane 0: pixels the group above is known to have published
    unsigned long long cseen = 0; // group 0, lane 0: the band above's progress word as last read
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
            if (g == 0 && p.carry_in == nullptr) {
#pragma unroll
                for (int c = 0; c < C; ++c) din[c] = 0.0f;
            } else if (g == 0) {
                if (p.carry_in_prog != nullptr && !errd_carry_ready(cseen, p.seq, pix)) {
                    long long spins = 0;
                    while (!errd_carry_ready(cseen = *reinterpret_cast<const volatile unsigned long long*>(p.carry_in_prog),
                                             p.seq, pix)) {
                        if (++spins > (1ll << 31)) __trap(); // the band above never delivered: fail instead of hanging
                        __nanosleep(64);
                    }
                    __threadfence_system();
                }
#pragma unroll
                for (int c = 0; c < C; ++c) din[c] = __ldcv(p.carry_in + (size_t)pix * C + c);
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
        if (carry) {
            const int q = (on && pix >= 1) ? pix - 1 : ((pix == W) ? W - 1 : -1);
            if (q >= 0) {
#pragma unroll
                for (int c = 0; c < C; ++c) p.carry_out[(size_t)q * C + c] = dn[c];
                // (every 32 pixels and the last: one system-scope fence per 32 peer stores)
                if (p.carry_out_prog != nullptr && ((q & 31) == 31 || q == W - 1)) {
                    __threadfence_system();
                    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p.carry_out_prog),
                                 "l"(((unsigned long long)p.seq << 32) | (unsigned)(q + 1)) : "memory");
                }
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
int errd_groups(int rows) { return (rows + 31) / 32; }

// The workspace of one call: byte offsets of its segments, in this order, each 256-byte aligned.
// A call covers src_rows x src_cols source pixels, mid_rows x dst_cols intermediate pixels and
// dst_rows x dst_cols destination pixels (the whole image, a shard's band or a window and its footprint).
//   mid        the intermediate: mid_rows rows of mid_pitch(dst_cols) floats (at offset 0)
//   in32       float copy of a double source
//   out32      float copy of the destination (double output, error diffusion)
//   errd_bnd   error diffusion: boundary rows, one per 32-row group of the call's destination rows
//   errd_prog  error diffusion: progress counters
//   errd_carry error diffusion, shards only: the D rows received from the band above and sent to the band
//              below when they travel through NCCL (the mailbox schedules carry them in the mailbox)
//   src4       the widened source      } widened plans (pad4) only
//   dst4       the widened destination }
// Segments a plan does not use are empty (windows refuse error diffusion).
struct WsLayout {
    size_t in32, out32, errd_bnd, errd_prog, errd_carry, src4, dst4, total;
};
WsLayout ws_layout(const avirb200_plan* pl, int mid_rows, int src_rows, int dst_rows, bool shard, int src_cols,
                   int dst_cols) {
    const avirb200_plan_desc& d = pl->desc;
    const bool f64_in = pl->io_in_type == AVIRB200_F64;
    const bool f32_out = pl->io_out_type == AVIRB200_F64 || pl->errd;
    WsLayout w;
    size_t off = align_up((size_t)mid_rows * mid_pitch(pl, dst_cols) * sizeof(float), 256);
    auto seg = [&](bool on, size_t bytes) {
        const size_t at = off;
        if (on) off += align_up(bytes, 256);
        return at;
    };
    w.in32 = seg(f64_in, (size_t)src_cols * src_rows * d.channels * sizeof(float));
    w.out32 = seg(f32_out, (size_t)dst_cols * dst_rows * d.channels * sizeof(float));
    w.errd_bnd = seg(pl->errd, (size_t)errd_groups(dst_rows) * d.dst_w * d.channels * sizeof(float));
    w.errd_prog = seg(pl->errd, (size_t)errd_groups(dst_rows) * sizeof(int));
    w.errd_carry = seg(pl->errd && shard, 2 * (size_t)d.dst_w * d.channels * sizeof(float));
    w.src4 = seg(pl->pad4, (size_t)src_rows * src_cols * 4 * elem_size(d.in_type));
    w.dst4 = seg(pl->pad4, (size_t)dst_rows * dst_cols * 4 * elem_size(d.out_type));
    w.total = off;
    return w;
}
// The whole image's layout (resize_device, the per-pass entry points, the banded host call).
WsLayout ws_layout(const avirb200_plan* pl) {
    const avirb200_plan_desc& d = pl->desc;
    return ws_layout(pl, d.src_h, d.src_h, d.dst_h, false, d.src_w, d.dst_w);
}
// One band of the sharded schedule.
WsLayout ws_layout(const avirb200_plan* pl, const avirb200_shard_info& si) {
    return ws_layout(pl, si.need_rows, si.src_rows, si.dst_rows, true, pl->desc.src_w, pl->desc.dst_w);
}
// A destination window of w columns and h rows with its footprint wi.
WsLayout ws_layout(const avirb200_plan* pl, const avirb200_window_info& wi, int w, int h) {
    return ws_layout(pl, wi.mid_rows, wi.src_h, h, false, wi.src_w, w);
}

// A double source's rows (cols pixels each) as floats into the workspace's in32: upstream's (float) cast.
int narrow_source(const avirb200_plan* pl, const void* d_src, size_t src_pitch, int cols, int rows, float* in32,
                  cudaStream_t st, int* launches) {
    const int re = cols * pl->desc.channels;
    const long long n = (long long)re * rows;
    if (n == 0) return 0;
    narrow_f64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(static_cast<const double*>(d_src), (long long)src_pitch,
                                                                   in32, re, rows);
    ++*launches;
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// Where a band's ditherer takes the D row of its first row from and leaves the D row below its last (ErrdParams).
struct ErrdCarry {
    const float* in = nullptr;
    const unsigned long long* in_prog = nullptr;
    float* out = nullptr;
    unsigned long long* out_prog = nullptr;
    unsigned seq = 0;
};

// The column pass's float rows (out32: rows x cols pixels) into the caller's destination: widened to double,
// or dithered (whole rows: cols is the image's width) with the boundary rows and counters at bnd / prog.
int finish_rows(const avirb200_plan* pl, const float* out32, float* bnd, int* prog, int cols, int rows, void* d_dst,
                size_t dst_pitch, const ErrdCarry& carry, cudaStream_t st, int* launches) {
    const avirb200_plan_desc& d = pl->desc;
    if (pl->io_out_type == AVIRB200_F64) {
        const int re = cols * d.channels;
        const long long n = (long long)re * rows;
        if (n == 0) return 0;
        widen_f32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(out32, static_cast<double*>(d_dst),
                                                                      (long long)dst_pitch, re, rows);
        ++*launches;
        CUDA_TRY(cudaGetLastError());
    }
    if (pl->errd) {
        ErrdParams ep;
        ep.src = out32;
        ep.dst = d_dst;
        ep.dst_pitch = (long long)dst_pitch;
        ep.W = cols; ep.H = rows;
        ep.dst_type = pl->io_out_type;
        ep.round_mode = d.round_mode;
        ep.planar = (d.sum_mode == AVIRB200_SUM_DIL8) ? 1 : 0;
        ep.tr_mul = d.tr_mul; ep.tr_mul_inv = d.tr_mul_inv; ep.pk_out = d.pk_out;
        ep.boundary = bnd;
        ep.progress = prog;
        ep.carry_in = carry.in; ep.carry_in_prog = carry.in_prog;
        ep.carry_out = carry.out; ep.carry_out_prog = carry.out_prog;
        ep.seq = carry.seq;
        const int groups = errd_groups(rows);
        CUDA_TRY(cudaMemsetAsync(prog, 0, (size_t)groups * 4, st));
        switch (d.channels) {
        case 1: errd_kernel<1><<<groups, 32, 0, st>>>(ep); break;
        case 2: errd_kernel<2><<<groups, 32, 0, st>>>(ep); break;
        case 3: errd_kernel<3><<<groups, 32, 0, st>>>(ep); break;
        default: errd_kernel<4><<<groups, 32, 0, st>>>(ep); break;
        }
        ++*launches;
        CUDA_TRY(cudaGetLastError());
    }
    return 0;
}

// ---- banded host calls: pageable images through page-locked bounce buffers ------------------------

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
// Error diffusion: band q-1's ditherer stores the D row below its last row into band q's mailbox with peer
// stores and raises a progress word (call sequence number << 32 | pixels published); band q's ditherer waits
// on it pixel by pixel.  The word names its call, so it is never reset (DESIGN.md section 7).
//
// The mailbox of band q, as MailboxLayout describes it:
//   [256 B header: flag "from above" at +0, flag "from below" at +4, the sender's counters at +64,
//    the error-diffusion progress words of slots 0 and 1 at +128 and +136]
//   slot 0: [rows from q-1: halo_up(q)] [rows from q+1: halo_down(q), at +align256(up_bytes)]
//           [error diffusion: D row from q-1, dst_w * channels floats, at +align256(up) + align256(down)]
//   slot 1: the same
struct MailboxLayout {
    static constexpr size_t kHeader = 256, kCounters = 64, kErrdProgress = 128;
    size_t up_bytes = 0, down_bytes = 0, errd_bytes = 0;
    MailboxLayout() = default;
    MailboxLayout(const avirb200_plan* pl, const avirb200_shard_info& si)
        : up_bytes((size_t)si.halo_up * mid_pitch(pl) * sizeof(float)),
          down_bytes((size_t)si.halo_down * mid_pitch(pl) * sizeof(float)),
          errd_bytes(pl->errd ? (size_t)pl->desc.dst_w * pl->desc.channels * sizeof(float) : 0) {}
    size_t slot_bytes() const { return align_up(up_bytes, 256) + align_up(down_bytes, 256) + align_up(errd_bytes, 256); }
    size_t bytes(int slots) const { return kHeader + (size_t)slots * slot_bytes(); }
    // the mailbox at `box` (this process's address of it), slot `slot`
    avs::StreamMailbox at(char* box, int slot) const {
        char* s = box + kHeader + (size_t)slot * slot_bytes();
        return {reinterpret_cast<float*>(s), reinterpret_cast<float*>(s + align_up(up_bytes, 256)),
                reinterpret_cast<unsigned*>(box), reinterpret_cast<unsigned long long*>(box + kCounters)};
    }
    // error diffusion: the D row from the band above and its progress word, slot `slot`
    float* errd_row(char* box, int slot) const {
        return reinterpret_cast<float*>(box + kHeader + (size_t)slot * slot_bytes() + align_up(up_bytes, 256) +
                                        align_up(down_bytes, 256));
    }
    unsigned long long* errd_progress(char* box, int slot) const {
        return reinterpret_cast<unsigned long long*>(box + kErrdProgress) + slot;
    }
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

// Sharded calls: after the row pass (stream st) the band's boundary rows go to the neighbours' mailboxes on
// the exchange stream (copy engines), each followed by the call's sequence number (at `word`).
int sharded_push(avirb200_plan* pl, cudaStream_t st, const float* own, const avs::StreamLink& l, const unsigned* word) {
    const size_t rowf = mid_pitch(pl), rowb = rowf * sizeof(float);
    const int top_rows = avs::stream_rows_up(l), bot_rows = avs::stream_rows_down(l);
    PeerExchange& x = pl->x;
    int r = x.fork(st);
    if (r == 0 && top_rows > 0)
        r = push_rows(l.above.from_dn, rowb, own, rowb, rowb, top_rows, &l.above.flags[1], word, x.stream);
    if (r == 0 && bot_rows > 0)
        r = push_rows(l.below.from_up, rowb, own + (size_t)(l.me->src_rows - bot_rows) * rowf, rowb, rowb, bot_rows,
                      &l.below.flags[0], word, x.stream);
    return r;
}

// Plans the banded host call runs unbanded: double buffers and error diffusion (bands on one compute stream would
// restart the ditherer's wavefront once per band).
// The plan's element types: the caller's (io_*), and what the kernels read and write (desc).
void set_plan_types(avirb200_plan* pl, const avirb200_plan_desc* desc) {
    pl->desc = *desc;
    pl->io_in_type = desc->in_type;
    pl->io_out_type = desc->out_type;
    pl->mid_ch = desc->channels;
    if (desc->in_type == AVIRB200_F64) pl->desc.in_type = AVIRB200_F32;   // cast on the device first
    if (desc->out_type == AVIRB200_F64) pl->desc.out_type = AVIRB200_F32; // widened on the device last
    if (desc->dither == 1 && (desc->out_type == AVIRB200_U8 || desc->out_type == AVIRB200_U16)) {
        // the column pass delivers the gamma-corrected float rows; errd_kernel rounds them in row order
        pl->errd = true;
        pl->desc.out_type = AVIRB200_F32;
    }
}

bool plan_has_f64(const avirb200_plan* pl) {
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
    set_plan_types(pl.get(), desc);
    if (pl->errd) {
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
    {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, pl->device) == cudaSuccess && n > 0)
            pl->sm_count = n;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMaxSharedMemoryPerBlockOptin, pl->device) == cudaSuccess && n > 0)
            pl->smem_optin = (size_t)n;
    }
    // The generic kernel runs every pass no other kernel takes (and every pass under KERNEL_FAMILY 1), so a
    // plan whose pass does not fit it even as one output of one line per block is refused here, before any
    // launch.  What remains are long lines to very few pixels: a 4-channel line of more than about 11 600
    // source pixels to one pixel on an H100 (the source span of that one output, 5 floats per position).
    pl->cfg_h = choose_generic_config(host_axis_view(pl->h.desc), desc->channels, 0, desc->dst_w, pl->smem_optin);
    pl->cfg_v = choose_generic_config(host_axis_view(pl->v.desc), desc->channels, 0, desc->dst_h, pl->smem_optin);
    for (int a = 0; a < 2; ++a) {
        const PassConfig& c = a ? pl->cfg_v : pl->cfg_h;
        if (c.smem > pl->smem_optin)
            return fail(AVIRB200_ERR_UNSUPPORTED,
                        std::string(a ? "column pass" : "row pass") + ": one output of one line needs " +
                            std::to_string(c.smem) + " bytes of shared memory, more than the " +
                            std::to_string(pl->smem_optin) + " a block of this device can have");
    }

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
    *out = pl.release();
    return 0;
}

void avirb200_plan_destroy(avirb200_plan* pl) {
    if (pl == nullptr) return;
    cudaFree(pl->arena);
    fast_plan_free(pl->fast);
    pl->x.close();
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

int avirb200_plan_last_launches(const avirb200_plan* pl) {
    return pl ? pl->last_launches.load(std::memory_order_relaxed) : 0;
}

} // extern "C"

namespace {

// The whole image (win null), or the destination window [x0, x0 + w) x [y0, y0 + h) with its footprint
// *win: d_src holds the footprint, d_dst receives the window.  *n_launches (when given): the call's launches.
int resize_region(const avirb200_plan* pl, const avirb200_window_info* win, int x0, int y0, int w, int h,
                  const void* d_src, size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws, void* stream,
                  int* n_launches = nullptr) {
    const avirb200_plan_desc& d = pl->desc;
    const int src_w = win ? win->src_w : d.src_w, src_h = win ? win->src_h : d.src_h;
    if (src_pitch < (size_t)src_w * d.channels || dst_pitch < (size_t)w * d.channels)
        return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    if (const int e = check_device(pl->device)) return e;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int launches = 0;
    char* wsb = static_cast<char*>(d_ws);
    const WsLayout ws = win ? ws_layout(pl, *win, w, h) : ws_layout(pl);
    float* in32 = reinterpret_cast<float*>(wsb + ws.in32);
    float* out32 = reinterpret_cast<float*>(wsb + ws.out32);
    const void* ksrc = d_src;
    size_t ksrc_pitch = src_pitch;
    void* kdst = d_dst;
    size_t kdst_pitch = dst_pitch;
    if (pl->io_in_type == AVIRB200_F64) {
        const int e = narrow_source(pl, d_src, src_pitch, src_w, src_h, in32, st, &launches);
        if (e != 0) return e;
        ksrc = in32;
        ksrc_pitch = (size_t)src_w * d.channels;
    }
    if (pl->io_out_type == AVIRB200_F64 || pl->errd) {
        kdst = out32;
        kdst_pitch = (size_t)w * d.channels;
    }
    // (a window: the intermediate columns [x0, x0 + w) from its footprint's source columns, and the column
    // pass over those columns only)
    float* mid = static_cast<float*>(d_ws);
    PassRequest row = row_request(d, ksrc, ksrc_pitch, src_h, mid, mid_pitch(pl, w));
    const int mid_lo = win ? win->mid_row0 : 0, mid_hi = win ? win->mid_row0 + win->mid_rows : d.src_h;
    PassRequest col = col_request(d, w, mid, mid_pitch(pl, w), mid_lo, mid_hi, kdst, kdst_pitch, y0, y0 + h);
    if (win != nullptr) {
        row.out0 = row.dst_base = x0;
        row.out1 = x0 + w;
        row.src_base = row.src_lo = win->src_x0;
        row.src_hi = win->src_x0 + win->src_w;
    }
    row.scratch4 = wsb + ws.src4;
    col.scratch4 = wsb + ws.dst4;
    int r = run_pass(pl, row, st, &launches);
    if (r == 0) r = run_pass(pl, col, st, &launches);
    if (r == 0)
        r = finish_rows(pl, out32, reinterpret_cast<float*>(wsb + ws.errd_bnd), reinterpret_cast<int*>(wsb + ws.errd_prog), w,
                        h, d_dst, dst_pitch, ErrdCarry(), st, &launches);
    pl->last_launches.store(launches, std::memory_order_relaxed);
    if (n_launches != nullptr) *n_launches = launches;
    return r;
}

} // namespace

extern "C" {

int avirb200_resize_device(const avirb200_plan* pl, const void* d_src, size_t src_pitch, void* d_dst,
                           size_t dst_pitch, void* d_ws, void* stream) {
    if (pl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    return resize_region(pl, nullptr, 0, 0, pl->desc.dst_w, pl->desc.dst_h, d_src, src_pitch, d_dst, dst_pitch, d_ws,
                         stream);
}

int avirb200_window_query(const avirb200_plan* pl, int x0, int y0, int w, int h, avirb200_window_info* info) {
    if (pl == nullptr || info == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    return window_compute(pl, x0, y0, w, h, info);
}

int avirb200_window_query_desc(const avirb200_plan_desc* desc, int x0, int y0, int w, int h,
                               avirb200_window_info* info) {
    if (desc == nullptr || info == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (desc->h.nsteps < 1 || desc->h.nsteps > AVIRB200_MAX_STEPS || desc->v.nsteps < 1 ||
        desc->v.nsteps > AVIRB200_MAX_STEPS)
        return fail(AVIRB200_ERR_BAD_ARG, "axis: nsteps out of range");
    // (as avirb200_plan_create decides it)
    const bool errd = desc->dither == 1 && (desc->out_type == AVIRB200_U8 || desc->out_type == AVIRB200_U16);
    return window_compute(host_axis_view(desc->h), host_axis_view(desc->v), errd, x0, y0, w, h, info);
}

int avirb200_window_workspace_bytes(const avirb200_plan* pl, int x0, int y0, int w, int h, size_t* bytes) {
    if (pl == nullptr || bytes == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_window_info wi;
    const int r = window_compute(pl, x0, y0, w, h, &wi);
    if (r != 0) return r;
    *bytes = ws_layout(pl, wi, w, h).total;
    return 0;
}

int avirb200_resize_window_device(const avirb200_plan* pl, int x0, int y0, int w, int h, const void* d_src,
                                  size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws, void* stream) {
    if (pl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_window_info wi;
    const int r = window_compute(pl->h.hostdev, pl->v.hostdev, pl->errd, x0, y0, w, h, &wi);
    if (r != 0) return r;
    return resize_region(pl, &wi, x0, y0, w, h, d_src, src_pitch, d_dst, dst_pitch, d_ws, stream);
}

int avirb200_resize_window_host(avirb200_plan* pl, int x0, int y0, int w, int h, const void* h_src,
                                size_t src_pitch, void* h_dst, size_t dst_pitch) {
    if (pl == nullptr || h_src == nullptr || h_dst == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    avirb200_window_info wi;
    const int r = window_compute(pl->h.hostdev, pl->v.hostdev, pl->errd, x0, y0, w, h, &wi);
    if (r != 0) return r;
    // the footprint only; the whole source is read before any destination pixel is written (aliasing)
    const size_t C = d.channels;
    const HostRect src = host_rect(h_src, src_pitch, d.src_w * C, elem_size(pl->io_in_type), wi.src_x0 * C, wi.src_w * C,
                                   wi.src_y0, wi.src_h);
    const HostRect dst = host_rect(h_dst, dst_pitch, w * C, elem_size(pl->io_out_type), 0, w * C, 0, h);
    return staged_call(pl->mx, staging_of(pl->device), pl->device, &pl->stream, src, dst, ws_layout(pl, wi, w, h).total,
                       [&](const void* s, void* o, void* ws, cudaStream_t st) {
                           // (the tile kernel's tables of the window's ranges, on the plan's device)
                           fast_prepare_columns(pl->fast, x0, x0 + w);
                           fast_prepare_range(pl->fast, y0, y0 + h);
                           return resize_region(pl, &wi, x0, y0, w, h, s, wi.src_w * C, o, w * C, ws, st);
                       });
}

int avirb200_row_pass_device(const avirb200_plan* pl, const void* d_src, size_t src_pitch,
                             void* d_ws, void* stream) {
    if (pl == nullptr || d_src == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const WsLayout ws = ws_layout(pl);
    int launches = 0;
    if (pl->io_in_type == AVIRB200_F64) { // the float copy of the source first, as resize_device makes it
        if (src_pitch < (size_t)d.src_w * d.channels) return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
        float* in32 = reinterpret_cast<float*>(static_cast<char*>(d_ws) + ws.in32);
        const int e = narrow_source(pl, d_src, src_pitch, d.src_w, d.src_h, in32, st, &launches);
        if (e != 0) return e;
        d_src = in32;
        src_pitch = (size_t)d.src_w * d.channels;
    }
    PassRequest q = row_request(d, d_src, src_pitch, d.src_h, static_cast<float*>(d_ws), mid_pitch(pl));
    q.scratch4 = static_cast<char*>(d_ws) + ws.src4;
    return run_pass(pl, q, st, &launches);
}

int avirb200_col_pass_device(const avirb200_plan* pl, const void* d_ws, void* d_dst,
                             size_t dst_pitch, void* stream) {
    if (pl == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* wsb = static_cast<char*>(const_cast<void*>(d_ws));
    const WsLayout ws = ws_layout(pl);
    int launches = 0;
    // double output and error diffusion: the float rows into the workspace, then widened / dithered
    const bool f32_out = pl->io_out_type == AVIRB200_F64 || pl->errd;
    if (f32_out && dst_pitch < (size_t)d.dst_w * d.channels) return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    float* out32 = reinterpret_cast<float*>(wsb + ws.out32);
    PassRequest q = col_request(d, d.dst_w, static_cast<const float*>(d_ws), mid_pitch(pl), 0, d.src_h,
                                f32_out ? static_cast<void*>(out32) : d_dst, f32_out ? (size_t)d.dst_w * d.channels : dst_pitch,
                                0, d.dst_h);
    q.scratch4 = wsb + ws.dst4;
    int r = run_pass(pl, q, st, &launches);
    if (r == 0 && f32_out)
        r = finish_rows(pl, out32, reinterpret_cast<float*>(wsb + ws.errd_bnd), reinterpret_cast<int*>(wsb + ws.errd_prog),
                        d.dst_w, d.dst_h, d_dst, dst_pitch, ErrdCarry(), st, &launches);
    return r;
}

int avirb200_resize_device_batch(const avirb200_plan* pl, int n, const void* const* d_srcs, size_t src_pitch,
                                 void* const* d_dsts, size_t dst_pitch, void* d_ws, void* stream) {
    if (pl == nullptr || d_srcs == nullptr || d_dsts == nullptr || d_ws == nullptr || n < 0)
        return fail(AVIRB200_ERR_BAD_ARG, "bad argument");
    int total = 0;
    for (int i = 0; i < n; ++i) {
        // frames share the workspace: the stream keeps frame i's column pass ahead of frame i+1's row pass
        if (d_srcs[i] == nullptr || d_dsts[i] == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
        int launches = 0;
        const int r = resize_region(pl, nullptr, 0, 0, pl->desc.dst_w, pl->desc.dst_h, d_srcs[i], src_pitch, d_dsts[i],
                                    dst_pitch, d_ws, stream, &launches);
        if (r != 0) return r;
        total += launches;
    }
    pl->last_launches.store(total, std::memory_order_relaxed);
    return 0;
}

int avirb200_resize_host(avirb200_plan* pl, const void* h_src, size_t src_pitch, void* h_dst,
                         size_t dst_pitch) {
    if (pl == nullptr || h_src == nullptr || h_dst == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    const size_t in_el = elem_size(pl->io_in_type), out_el = elem_size(pl->io_out_type);
    const size_t sw = (size_t)d.src_w * d.channels, dw = (size_t)d.dst_w * d.channels;
    const HostRect src = host_rect(h_src, src_pitch, sw, in_el, 0, sw, 0, d.src_h);
    const HostRect dst = host_rect(h_dst, dst_pitch, dw, out_el, 0, dw, 0, d.dst_h);
    const size_t in_row = src.row, out_row = dst.row;
    const size_t in_bytes = in_row * d.src_h, out_bytes = out_row * d.dst_h;
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
    if (plan_has_f64(pl)) nb = 1; // the casts and the ditherer run over the whole image
    std::vector<avirb200_shard_info> si;
    while (nb >= 2) { // fewer bands until every band's column pass needs only its neighbours' rows
        si.assign(nb, avirb200_shard_info());
        bool ok = true;
        for (int b = 0; b < nb && ok; ++b) ok = (shard_compute(pl, b, nb, &si[b]) == 0);
        if (ok) break;
        nb /= 2;
    }
    if (nb >= 2) {
        HostCall call(pl->mx, staging_of(pl->device));
        {
            const int r0 = call.begin(pl->device, &pl->stream, src, dst, ws_layout(pl).total);
            if (r0 != 0) return r0;
        }
        Staging& sg = call.sg;
        // the tile kernel's tables of the bands' destination rows (a launch does not build them)
        for (int b = 0; b < nb; ++b) fast_prepare_range(pl->fast, si[b].dst_row0, si[b].dst_row0 + si[b].dst_rows);
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
        char* src4 = static_cast<char*>(sg.d_ws) + ws_layout(pl).src4;
        char* dst4 = static_cast<char*>(sg.d_ws) + ws_layout(pl).dst4;
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
                CUDA_TRY(cudaMemcpyAsync(static_cast<char*>(sg.d_src) + (size_t)si[b].src_row0 * in_row, hs,
                                         (size_t)si[b].src_rows * in_row, cudaMemcpyHostToDevice, pl->stream_in));
                CUDA_TRY(cudaEventRecord(pl->ev_slot[slot], pl->stream_in));
                CUDA_TRY(cudaEventRecord(pl->ev_in[b], pl->stream_in));
                return 0;
            }
            CUDA_TRY(cudaMemcpy2DAsync(static_cast<char*>(sg.d_src) + (size_t)si[b].src_row0 * in_row, in_row,
                                       static_cast<const char*>(h_src) + (size_t)si[b].src_row0 * src_pitch * in_el,
                                       src_pitch * in_el, in_row, si[b].src_rows, cudaMemcpyHostToDevice,
                                       pl->stream_in));
            CUDA_TRY(cudaEventRecord(pl->ev_in[b], pl->stream_in));
            return 0;
        };
        { const int r0 = copy_in(0); if (r0 != 0) return r0; }
        auto col_band = [&](int b) -> int {
            char* dd = static_cast<char*>(sg.d_dst) + (size_t)si[b].dst_row0 * out_row;
            PassRequest q = col_request(d, d.dst_w, static_cast<const float*>(sg.d_ws), rowf, 0, d.src_h, dd, dw,
                                        si[b].dst_row0, si[b].dst_row0 + si[b].dst_rows);
            q.scratch4 = dst4 + (size_t)si[b].dst_row0 * dst4_row;
            const int r = run_pass(pl, q, pl->stream, &launches);
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
            PassRequest q = row_request(d, static_cast<const char*>(sg.d_src) + (size_t)si[b].src_row0 * in_row, sw,
                                        si[b].src_rows, static_cast<float*>(sg.d_ws) + (size_t)si[b].src_row0 * rowf, rowf);
            q.scratch4 = src4 + (size_t)si[b].src_row0 * src4_row;
            int r = run_pass(pl, q, pl->stream, &launches);
            if (r != 0) return r;
            if (b > 0 && (r = col_band(b - 1)) != 0) return r; // needs rows of bands b-2 .. b only
        }
        int r = col_band(nb - 1);
        if (r != 0) return r;
        pl->last_launches.store(launches, std::memory_order_relaxed);
        CUDA_TRY(cudaStreamSynchronize(pl->stream_out));
        CUDA_TRY(cudaStreamSynchronize(pl->stream));
        if (drainer.t.joinable()) drainer.t.join(); // the last bands reach the caller's memory
        return 0;
    }
    return staged_call(pl->mx, staging_of(pl->device), pl->device, &pl->stream, src, dst, ws_layout(pl).total,
                       [&](const void* s, void* o, void* ws, cudaStream_t st) {
                           return avirb200_resize_device(pl, s, sw, o, dw, ws, st);
                       });
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

int avirb200_shard_layout_desc(const avirb200_plan_desc* desc, int rank, int nranks, size_t* ws_bytes,
                               size_t* mailbox_bytes) {
    if (desc == nullptr || ws_bytes == nullptr || mailbox_bytes == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    if (desc->channels < 1 || desc->channels > 4 || desc->in_type < 0 || desc->in_type > 3 || desc->out_type < 0 ||
        desc->out_type > 3)
        return fail(AVIRB200_ERR_BAD_ARG, "bad image geometry or element type");
    if (desc->v.nsteps < 1 || desc->v.nsteps > AVIRB200_MAX_STEPS)
        return fail(AVIRB200_ERR_BAD_ARG, "axis: nsteps out of range");
    // (host arithmetic on a plan that holds only its types: ws_layout and MailboxLayout read nothing else)
    avirb200_plan pl;
    set_plan_types(&pl, desc);
    if (desc->channels < 4 && !plan_has_f64(&pl))
        return fail(AVIRB200_ERR_UNSUPPORTED, "shard layout from a descriptor: a 1..3-channel plan may run widened "
                                              "to 4 channels, which plan creation decides");
    avirb200_shard_info si;
    const int r = shard_compute_axis(host_axis_view(desc->v), rank, nranks, &si);
    if (r != 0) return r;
    *ws_bytes = ws_layout(&pl, si).total;
    *mailbox_bytes = MailboxLayout(&pl, si).bytes(2);
    return 0;
}

} // extern "C"

namespace {

// avirb200_resize_sharded; for nranks > 1 the caller holds pl->mx.
int sharded(avirb200_plan* pl, void* comm, int rank, int nranks, const void* d_src, size_t src_pitch, void* d_dst,
            size_t dst_pitch, void* d_ws, cudaStream_t st) {
    int r = check_device(pl->device);
    if (r != 0) return r;
    avirb200_shard_info si;
    r = shard_compute(pl, rank, nranks, &si);
    if (r != 0) return r;
    const avirb200_plan_desc& d = pl->desc;
    const size_t rowf = mid_pitch(pl);
    const size_t in_el = elem_size(d.in_type);
    float* mid = static_cast<float*>(d_ws);
    float* own = mid + (size_t)si.halo_up * rowf;
    const WsLayout ws = ws_layout(pl, si);
    char* wsb = static_cast<char*>(d_ws);
    char* src4 = wsb + ws.src4;
    char* dst4 = wsb + ws.dst4;
    const size_t src4_row = (size_t)d.src_w * 4 * in_el;
    int launches = 0;
    const bool f32_out = pl->io_out_type == AVIRB200_F64 || pl->errd;
    if (f32_out && dst_pitch < (size_t)d.dst_w * d.channels) return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    // Double buffers: the band's source rows as floats first.  Double output and error diffusion: the column
    // pass writes the band's float rows into the workspace, finish_rows() widens or dithers them last.
    if (pl->io_in_type == AVIRB200_F64) {
        if (src_pitch < (size_t)d.src_w * d.channels) return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
        float* in32 = reinterpret_cast<float*>(wsb + ws.in32);
        if ((r = narrow_source(pl, d_src, src_pitch, d.src_w, si.src_rows, in32, st, &launches)) != 0) return r;
        d_src = in32;
        src_pitch = (size_t)d.src_w * d.channels;
    }
    float* out32 = reinterpret_cast<float*>(wsb + ws.out32);
    auto finish = [&](const ErrdCarry& cy) {
        return finish_rows(pl, out32, reinterpret_cast<float*>(wsb + ws.errd_bnd), reinterpret_cast<int*>(wsb + ws.errd_prog),
                           d.dst_w, si.dst_rows, d_dst, dst_pitch, cy, st, &launches);
    };
    // the band's passes: its own rows into `own`, its destination rows from the intermediate rows it holds
    PassRequest row = row_request(d, d_src, src_pitch, si.src_rows, own, rowf);
    row.scratch4 = src4;
    PassRequest col = col_request(d, d.dst_w, mid, rowf, si.need_row0, si.need_row0 + si.need_rows,
                                  f32_out ? static_cast<void*>(out32) : d_dst,
                                  f32_out ? (size_t)d.dst_w * d.channels : dst_pitch, si.dst_row0, si.dst_row0 + si.dst_rows);
    col.scratch4 = dst4;
    if (nranks <= 1) {
        r = run_pass(pl, row, st, &launches);
        if (r == 0) r = run_pass(pl, col, st, &launches);
        if (r == 0 && f32_out) r = finish(ErrdCarry());
        pl->last_launches.store(launches, std::memory_order_relaxed);
        return r;
    }
    Nccl* nc = nullptr;
    if ((r = comm_nccl(comm, &nc)) != 0) return r;
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

    PeerExchange& x = pl->x;
    const MailboxLayout mine(pl, si), above(pl, up), below(pl, down);
    if (pl->opt_overlap && (r = x.open(comm, rank, nranks, mine.bytes(2), MailboxLayout::kHeader, st)) != 0) return r;
    if (pl->opt_overlap && x.usable) {
        const PeerExchange::Call call = x.next_call();
        const char* srcb = static_cast<const char*>(d_src);
        auto rows_pass = [&](int row0, int nrows) -> int {
            PassRequest q = row_request(d, srcb + (size_t)row0 * src_pitch * in_el, src_pitch, nrows,
                                        own + (size_t)row0 * rowf, rowf);
            q.scratch4 = src4 + (size_t)row0 * src4_row;
            return run_pass(pl, q, st, &launches);
        };
        const int need_up = (link.up && si.halo_up > 0) ? 1 : 0;
        const int need_down = (link.dn && si.halo_down > 0) ? 1 : 0;
        link.seq = call.seq;
        link.mine = mine.at(x.box, call.slot);
        if (link.up) link.above = above.at(x.box_up, call.slot);
        if (link.dn) link.below = below.at(x.box_down, call.slot);
        // AVIRB200_OPT_OVERLAP_HALO = 3, the fused exchange: the row kernel stores the rows the neighbours need
        // into their mailboxes as it produces them (peer stores over NVLink) and raises their flags when the
        // last of them is out; the column kernel reads the neighbours' rows in place from this rank's mailbox,
        // waiting on the flags only in the runs that touch them.  No exchange stream, no copy, no extra launch.
        // Either half falls back on its own (the mailbox protocol is the same): a row pass that is not on the
        // streaming kernel pushes with the copy engines, a column pass that is not pulls into the workspace.
        const bool fused = pl->opt_overlap == 3 && avs::stream_fused_rx_ok(link);
        const bool fused_tx = pl->opt_overlap == 3 && avs::stream_fused_tx_ok(link);
        bool pushed = false;
        if (fused_tx && top_rows + bot_rows > 0) {
            PassRequest q = row;
            const bool send = pass_family(pl, q).family == kFamilyStream;
            if (send) q.link = &link;
            if ((r = run_pass(pl, q, st, &launches)) != 0) return r;
            if (!send) { // (not on the streaming kernel: the copy engines push)
                if ((r = sharded_push(pl, st, own, link, call.word)) != 0) return r;
                pushed = true;
            }
        } else {
            // 1. the rows the neighbours need (one launch on the streaming kernel: two line segments),
            // 2. their push on the exchange stream, 3. the interior rows
            // (boundary rows first only on request, AVIRB200_OPT_OVERLAP_HALO = 2: the copy-engine push
            // of cfg3's 1.2 MB is short next to the extra launch the split costs)
            const bool split = pl->opt_overlap == 2 && top_rows + bot_rows < si.src_rows;
            if (split && !use_pad4(pl) && pass_family(pl, row).family == kFamilyStream) {
                PassRequest q = row;
                q.seg_top = top_rows;
                q.seg_bot = bot_rows;
                if (top_rows + bot_rows > 0 && (r = run_pass(pl, q, st, &launches)) != 0) return r;
            } else if (split) {
                if ((r = rows_pass(0, top_rows)) != 0) return r;
                if ((r = rows_pass(si.src_rows - bot_rows, bot_rows)) != 0) return r;
            } else if ((r = run_pass(pl, row, st, &launches)) != 0) {
                return r;
            }
            if ((r = sharded_push(pl, st, own, link, call.word)) != 0) return r;
            pushed = true;
            if (split && (r = rows_pass(top_rows, si.src_rows - top_rows - bot_rows)) != 0) return r;
        }
        // 4. the neighbours' rows: in place (fused), or wait for their sequence numbers and move them
        // mailbox -> workspace
        if (fused && (need_up || need_down) && pass_family(pl, col).family == kFamilyStream) {
            PassRequest q = col;
            q.link = &link;
            r = run_pass(pl, q, st, &launches);
        } else {
            if (need_up || need_down) {
                (void)cudaGetLastError();
                halo_pull_kernel<<<64, 256, 0, st>>>(link.mine.flags, call.seq, need_up, need_down,
                                                     reinterpret_cast<const float4*>(link.mine.from_up), reinterpret_cast<float4*>(mid),
                                                     need_up ? mine.up_bytes / 16 : 0,
                                                     reinterpret_cast<const float4*>(link.mine.from_dn),
                                                     reinterpret_cast<float4*>(own + (size_t)si.src_rows * rowf),
                                                     need_down ? mine.down_bytes / 16 : 0);
                ++launches;
                CUDA_TRY(cudaGetLastError());
            }
            r = run_pass(pl, col, st, &launches);
        }
        // 5. double output: widened; error diffusion: the D row of the band above from this rank's mailbox, the
        // band's own last D row into the mailbox of the rank below (peer stores), both in this call's slot
        // Two slots hold because the sender's column pass of call n+1 waits for the receiver's rows of call n+1,
        // which the receiver's stream produces after its ditherer of call n (DESIGN.md section 7).  A band that
        // needs no rows from below (halo_down 0) has no such wait: its D row goes through NCCL instead.
        if (r == 0 && f32_out) {
            ErrdCarry cy;
            cy.seq = call.seq;
            float* carry = reinterpret_cast<float*>(wsb + ws.errd_carry);
            const size_t rowd = (size_t)d.dst_w * d.channels;
            const bool in_box = link.up && up.halo_down > 0, out_box = link.dn && si.halo_down > 0;
            if (pl->errd && link.up) {
                if (in_box) {
                    cy.in = mine.errd_row(x.box, call.slot);
                    cy.in_prog = mine.errd_progress(x.box, call.slot);
                } else {
                    NCCL_TRY(nc->Recv(carry, rowd, 7, rank - 1, comm, st));
                    cy.in = carry;
                }
            }
            if (pl->errd && link.dn) {
                if (out_box) {
                    cy.out = below.errd_row(x.box_down, call.slot);
                    cy.out_prog = below.errd_progress(x.box_down, call.slot);
                } else {
                    cy.out = carry + rowd;
                }
            }
            r = finish(cy);
            if (r == 0 && pl->errd && link.dn && !out_box) NCCL_TRY(nc->Send(cy.out, rowd, 7, rank + 1, comm, st));
        }
        // the pushes read this call's workspace: the caller's stream does not end before them
        if (const int e = pushed ? x.join(st) : 0) return e;
        pl->last_launches.store(launches, std::memory_order_relaxed);
        return r;
    }
    // NCCL schedule: whole row pass, send/recv group, column pass, one stream
    if ((r = run_pass(pl, row, st, &launches)) != 0) return r;
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
    r = run_pass(pl, col, st, &launches);
    // error diffusion: the D row of the band above arrives once rank-1's ditherer is done, this band's goes to
    // rank+1 once its own is: the ranks' ditherers run one after another
    if (r == 0 && f32_out) {
        ErrdCarry cy;
        float* carry = reinterpret_cast<float*>(wsb + ws.errd_carry);
        const size_t rowd = (size_t)d.dst_w * d.channels;
        if (pl->errd && rank > 0) {
            NCCL_TRY(nc->Recv(carry, rowd, 7, rank - 1, comm, st));
            cy.in = carry;
        }
        if (pl->errd && rank + 1 < nranks) cy.out = carry + rowd;
        r = finish(cy);
        if (r == 0 && cy.out != nullptr) NCCL_TRY(nc->Send(cy.out, rowd, 7, rank + 1, comm, st));
    }
    pl->last_launches.store(launches, std::memory_order_relaxed);
    return r;
}

} // namespace

extern "C" {

int avirb200_resize_sharded(const avirb200_plan* cpl, void* comm, int rank, int nranks,
                            const void* d_src, size_t src_pitch, void* d_dst, size_t dst_pitch,
                            void* d_ws, void* stream) {
    if (cpl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    avirb200_plan* pl = const_cast<avirb200_plan*>(cpl); // (exchange state is created on first use)
    const cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (nranks <= 1) return sharded(pl, comm, rank, nranks, d_src, src_pitch, d_dst, dst_pitch, d_ws, st);
    std::lock_guard<std::mutex> lk(pl->mx);
    return sharded(pl, comm, rank, nranks, d_src, src_pitch, d_dst, dst_pitch, d_ws, st);
}

int avirb200_resize_sharded_host(avirb200_plan* pl, void* comm, int rank, int nranks, const void* h_src,
                                 size_t src_pitch, void* h_dst, size_t dst_pitch) {
    if (pl == nullptr || h_src == nullptr || h_dst == nullptr) return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    avirb200_shard_info si;
    const int r = shard_compute(pl, rank, nranks, &si);
    if (r != 0) return r;
    // (the caller's element types: double bands are staged as doubles, dithered ones as integers)
    const size_t sw = (size_t)d.src_w * d.channels, dw = (size_t)d.dst_w * d.channels;
    const HostRect src = host_rect(h_src, src_pitch, sw, elem_size(pl->io_in_type), 0, sw, 0, si.src_rows);
    const HostRect dst = host_rect(h_dst, dst_pitch, dw, elem_size(pl->io_out_type), 0, dw, 0, si.dst_rows);
    return staged_call(pl->mx, staging_of(pl->device), pl->device, &pl->stream, src, dst, ws_layout(pl, si).total,
                       [&](const void* s, void* o, void* ws, cudaStream_t st) {
                           // (the tile kernel's table of the band's rows, on the plan's device)
                           fast_prepare_range(pl->fast, si.dst_row0, si.dst_row0 + si.dst_rows);
                           return sharded(pl, comm, rank, nranks, s, sw, o, dw, ws, st);
                       });
}

int avirb200_resize_sharded_local(const avirb200_plan* pl, int nranks, const void* d_src,
                                  size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_ws,
                                  void* stream) {
    if (pl == nullptr || d_src == nullptr || d_dst == nullptr || d_ws == nullptr)
        return fail(AVIRB200_ERR_BAD_ARG, "null argument");
    const avirb200_plan_desc& d = pl->desc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t rowf = mid_pitch(pl);
    // (the caller's element types; the kernels' source is the band's float copy when it is double)
    const size_t in_el = elem_size(pl->io_in_type), out_el = elem_size(pl->io_out_type);
    const bool f64_in = pl->io_in_type == AVIRB200_F64, f32_out = pl->io_out_type == AVIRB200_F64 || pl->errd;
    if ((f64_in && src_pitch < (size_t)d.src_w * d.channels) || (f32_out && dst_pitch < (size_t)d.dst_w * d.channels))
        return fail(AVIRB200_ERR_BAD_ARG, "pitch smaller than a row");
    std::vector<avirb200_shard_info> si(nranks);
    std::vector<float*> mid(nranks), own(nranks);
    std::vector<PassRequest> row(nranks), col(nranks);
    std::vector<WsLayout> wsl(nranks);
    std::vector<char*> wsb(nranks);
    char* base = static_cast<char*>(d_ws);
    for (int r = 0; r < nranks; ++r) { // every band's segment: as avirb200_shard_workspace_bytes lays it out
        int e = shard_compute(pl, r, nranks, &si[r]);
        if (e != 0) return e;
        const WsLayout ws = wsl[r] = ws_layout(pl, si[r]);
        wsb[r] = base;
        mid[r] = reinterpret_cast<float*>(base);
        own[r] = mid[r] + (size_t)si[r].halo_up * rowf;
        const char* band_src = static_cast<const char*>(d_src) + (size_t)si[r].src_row0 * src_pitch * in_el;
        char* band_dst = static_cast<char*>(d_dst) + (size_t)si[r].dst_row0 * dst_pitch * out_el;
        row[r] = f64_in ? row_request(d, base + ws.in32, (size_t)d.src_w * d.channels, si[r].src_rows, own[r], rowf)
                        : row_request(d, band_src, src_pitch, si[r].src_rows, own[r], rowf);
        row[r].scratch4 = base + ws.src4;
        col[r] = col_request(d, d.dst_w, mid[r], rowf, si[r].need_row0, si[r].need_row0 + si[r].need_rows,
                             f32_out ? base + ws.out32 : band_dst, f32_out ? (size_t)d.dst_w * d.channels : dst_pitch,
                             si[r].dst_row0, si[r].dst_row0 + si[r].dst_rows);
        col[r].scratch4 = base + ws.dst4;
        base += ws.total;
    }
    int launches = 0;
    // double buffers: every band's source rows as floats (upstream's cast), before the row passes
    for (int r = 0; r < nranks && f64_in; ++r) {
        const int e = narrow_source(pl, static_cast<const char*>(d_src) + (size_t)si[r].src_row0 * src_pitch * in_el,
                                    src_pitch, d.src_w, si[r].src_rows, reinterpret_cast<float*>(wsb[r] + wsl[r].in32), st,
                                    &launches);
        if (e != 0) return e;
    }
    // The fused halo exchange of avirb200_resize_sharded (AVIRB200_OPT_OVERLAP_HALO = 3), with every band's
    // mailbox (one slot) in this device's memory: the same two kernels, parameters and protocol as between
    // ranks.  Only when every band may run both fused halves and both its passes run on the streaming kernel.
    // Error diffusion hands each band's last D row to the next band through the same mailboxes on every
    // schedule (the bands' ditherers run in stream order: no wait ever spins).
    std::vector<avs::StreamLink> link(nranks);
    std::vector<MailboxLayout> box(nranks);
    std::vector<size_t> box_off(nranks + 1, 0);
    bool fused = pl->opt_overlap == 3 && nranks > 1;
    for (int r = 0; r < nranks; ++r) {
        link[r].me = &si[r];
        if (r > 0) link[r].up = &si[r - 1];
        if (r + 1 < nranks) link[r].dn = &si[r + 1];
        fused = fused && avs::stream_fused_tx_ok(link[r]) && pass_family(pl, row[r]).family == kFamilyStream &&
                pass_family(pl, col[r]).family == kFamilyStream;
        box[r] = MailboxLayout(pl, si[r]);
        box_off[r + 1] = box_off[r] + box[r].bytes(1);
    }
    // the bands' float rows into the destination: widened, or dithered with the D row carried band to band
    auto finish_bands = [&](char* boxes) -> int {
        for (int r = 0; r < nranks && f32_out; ++r) {
            ErrdCarry cy;
            cy.seq = 1; // (the mailboxes are this call's own)
            if (pl->errd && r > 0) {
                cy.in = box[r].errd_row(boxes + box_off[r], 0);
                cy.in_prog = box[r].errd_progress(boxes + box_off[r], 0);
            }
            if (pl->errd && r + 1 < nranks) {
                cy.out = box[r + 1].errd_row(boxes + box_off[r + 1], 0);
                cy.out_prog = box[r + 1].errd_progress(boxes + box_off[r + 1], 0);
            }
            const int e = finish_rows(pl, reinterpret_cast<const float*>(wsb[r] + wsl[r].out32),
                                      reinterpret_cast<float*>(wsb[r] + wsl[r].errd_bnd),
                                      reinterpret_cast<int*>(wsb[r] + wsl[r].errd_prog), d.dst_w, si[r].dst_rows,
                                      static_cast<char*>(d_dst) + (size_t)si[r].dst_row0 * dst_pitch * out_el, dst_pitch,
                                      cy, st, &launches);
            if (e != 0) return e;
        }
        return 0;
    };
    char* boxes = nullptr;
    if (fused || (pl->errd && nranks > 1)) {
        CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&boxes), box_off[nranks], st));
        int e = 0;
        for (int r = 0; r < nranks && e == 0; ++r)
            if (cudaMemsetAsync(boxes + box_off[r], 0, MailboxLayout::kHeader, st) != cudaSuccess)
                e = fail(AVIRB200_ERR_CUDA, "sharded_local: mailbox header");
        if (e != 0) {
            cudaFreeAsync(boxes, st);
            return e;
        }
    }
    if (fused) {
        int e = 0;
        for (int r = 0; r < nranks; ++r) {
            link[r].mine = box[r].at(boxes + box_off[r], 0);
            link[r].seq = 1;
        }
        for (int r = 0; r < nranks; ++r) {
            if (r > 0) link[r].above = link[r - 1].mine;
            if (r + 1 < nranks) link[r].below = link[r + 1].mine;
            if (avs::stream_rows_up(link[r]) + avs::stream_rows_down(link[r]) > 0) row[r].link = &link[r];
            col[r].link = &link[r];
        }
        for (int r = 0; r < nranks && e == 0; ++r) e = run_pass(pl, row[r], st, &launches);
        for (int r = 0; r < nranks && e == 0; ++r) e = run_pass(pl, col[r], st, &launches);
        if (e == 0) e = finish_bands(boxes);
        cudaFreeAsync(boxes, st);
        pl->last_launches.store(launches, std::memory_order_relaxed);
        return e;
    }
    // (error diffusion: the mailboxes are released on every exit below)
    struct BoxGuard {
        char* p; cudaStream_t st;
        ~BoxGuard() { if (p != nullptr) cudaFreeAsync(p, st); }
    } box_guard{boxes, st};
    for (int r = 0; r < nranks; ++r) { // every band's row pass
        int e = run_pass(pl, row[r], st, &launches);
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
        int e = run_pass(pl, col[r], st, &launches);
        if (e != 0) return e;
    }
    if (const int e = finish_bands(boxes)) return e;
    pl->last_launches.store(launches, std::memory_order_relaxed);
    return 0;
}

} // extern "C"
