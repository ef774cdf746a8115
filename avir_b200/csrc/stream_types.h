// stream_types.h -- kernel parameters and host-side planning of the warp-streaming pass
// kernel (stream_kernel.cuh): decides whether an axis of a plan is one of the regular chains
// the kernel is instantiated for and folds the resize step's single effective phase into
// kernel-parameter taps.  Pure host code without CUDA calls: the engine (engine.cu) and the
// lockstep emulation used by the CPU tests (tests/emul) share it.
#pragma once

#include <stdint.h>
#include <string.h>

#include "avirb200.h"
#include "device_plan.h"
#include "pass_request.h"

namespace avs {

constexpr int kMaxSteps = 3;
constexpr int kLines = 16; // lines per warp (2 lanes per line): the 16-line strips of a pass
// Source code of the row pass beyond the plain element types: u8 pixels linearised on the way
// in (sRGB table for the colour channels, (float) b * InGammaMult for alpha; avir.h:2843-2931).
constexpr int kSrcU8Srgb = 4;
enum { K_FIR = 0, K_RESIZE = 1, K_RESIZE2 = 2, K_NONE = 3 };

// Run-time description of one step (kernel parameters: taps are constant-bank operands).
// A tap is stored as the pair (t, t): one operand of the packed two-lane multiply
// (mul.rn.f32x2, a lane pair = the two channels a thread owns).  taps[kTapOne] = (1, 1) is
// the multiplier of the packed add, see f2add() in stream_kernel.cuh.
constexpr int kTapOne = 64;
struct StreamTap {
    float lo, hi;
};
struct StreamStep {
    int out_len, in_len;
    int edge, latency;  // FIR
    int sp_first;       // RESIZE/RESIZE2: source position of output 0 (position j: sp_first + ADV*j)
    int zero_start;
    StreamTap taps[kTapOne + 1];
};

struct StreamParams {
    StreamStep s[kMaxSteps];
    int n_lines;          // rows (row pass) or pixel columns (column pass)
    // Two line segments in one launch (the rows a sharded call's neighbours need: the band's first
    // seg_a lines and its last seg_b lines, each cut into its own 16-line strips): seg_b > 0 turns it on;
    // the lines are 0 .. seg_a - 1 and seg_b_line0 .. seg_b_line0 + seg_b - 1 of the buffers.
    int seg_a, seg_b, seg_b_line0;
    int src_len;          // positions of the source line
    int out0, out1;       // final outputs [out0, out1) to produce
    const void* src;      // 4 interleaved channels; fp32, or (row pass) the caller's u8 / u16 pixels
    int src_type;         // AVIRB200_F32 / _U8 / _U16 / kSrcU8Srgb: selects the kernel instantiation (row pass)
    const float* srgb_lut; // kSrcU8Srgb: upstream's 256-entry linearisation table (device memory)
    float in_gamma_mult;   // kSrcU8Srgb: multiplier of the alpha channel
    long long src_pitch;  // elements between rows
    // Global source position held by the buffer's position 0: column pass, the intermediate row of a
    // shard's or a window's first row; row pass, the source column of a window's footprint's first column.
    int src_row_base;
    // Source positions the buffer actually holds, [src_lo, src_hi) (the whole line, a shard's band of
    // intermediate rows or a window's footprint columns).  A run starts and ends on round boundaries, so
    // its first / last round may compute outputs outside [out0, out1) (never stored) whose windows reach
    // past the band: reads clamp to this range, not just to the line.
    int src_lo, src_hi;
    void* dst;
    long long dst_pitch;
    int dst_type;
    int dst_row_base;     // final output stored at the destination's position 0 (row, or row-pass column)
    // the pixel stage (avb::PixelStage) in the order the kernel's parameter space has always held it
    int gamma_out, alpha_index;
    float out_gamma_mult;
    int round_mode;
    float tr_mul, tr_mul_inv, pk_out;
    // ---- fused halo exchange of sharded calls (engine.cu: AVIRB200_OPT_OVERLAP_HALO = 3) -----------
    // Row pass (sender): lines [0, xs_top) of the band are ALSO stored into the mailbox of the rank
    // above (xs_up_dst: its row 0), lines [xs_bot0, xs_bot0 + xs_bot) into the mailbox of the rank
    // below (xs_dn_dst); a warp that finishes a run over such lines adds its rounds to xs_count[0 / 1]
    // (this rank's memory, zero between calls; the total to reach is xs_units[..] strips x the rounds
    // of a strip), and the warp that completes the total zeroes the counter and writes xs_seq to the
    // neighbour's flag.  Null pointers: off.
    float* xs_up_dst;
    float* xs_dn_dst;
    unsigned* xs_up_flag;
    unsigned* xs_dn_flag;
    unsigned long long* xs_count;
    unsigned long long xs_units[2];
    unsigned xs_seq;
    int xs_top, xs_bot0, xs_bot;
    // Column pass (receiver): source rows below xr_own_lo come from xr_up_src (row need_row0 first),
    // rows from xr_own_hi on from xr_dn_src (row xr_own_hi first) -- the mailbox, read in place; a run
    // that touches them first waits for xr_flags[0 / 1] >= xr_seq.  xr_flags null: off.
    const float* xr_up_src;
    const float* xr_dn_src;
    const volatile unsigned* xr_flags;
    unsigned xr_seq;
    int xr_own_lo, xr_own_hi;
    // column pass, scheduling variant 2: CUtensorMap over the intermediate buffer (2-D, fp32:
    // n_lines * 4 elements per row, rows from p.src on; box 64 elements x SRC_N rows), encoded by
    // the launcher (stream_chain.cu)
    alignas(64) unsigned char tmap[128];
};

enum StreamChainId {
    kChainNone = 0,
    kChainDil24, // RESIZE(24, D2) -> FIR8                 cfg3, float8_dil mirror (k = 2)
    kChainInl24, // RESIZE(24, D2) -> FIR7                 k = 2, build mode 1, interleaved classes
    kChainInl3,  // FIR7 -> RESIZE(18, D2) -> FIR7         cfg3, float4 mirror (k = 2, build mode 0)
    kChainInl3D, // FIR15/2 -> RESIZE(18, D2) -> FIR7      cfg4 (k = 4, build mode 0)
    kChainDil56, // RESIZE(56, D4) -> FIR8                 cfg5, float8_dil mirror (k = 4, build mode 1)
    kChainUp2,   // FIR7 -> RESIZE2(24)                    cfg2 (k = 0.5, build mode 1)
    kChainDil24Q, // = kChainDil24 in 4-output batches, three warps per scheduler (selected instead of it
                  //   with AVIRB200_OPT_ALL_STREAM_CHAINS = 2)
    kChainCount
};

// Scheduling variants (same arithmetic; ChainC MODE in stream_kernel.cuh):
//   0  ring windows: every batch reads its whole window from the per-warp shared-memory rings
//   1  register windows: in the interior of a run the windows slide through registers, shared
//      memory carries the source ring only (each input read once)
//   2  = 1 with the column pass's source ring filled by one lane's tensor copies (TMA,
//      cp.async.bulk.tensor.2d) and tracked by mbarriers instead of per-lane cp.async groups
//      (the row pass runs 1)
//   3  = 0 without the straight-line loop for the interior rounds (every round takes the
//      checked path: the cross-check of the other three)
constexpr int kStreamVariants = 4;
// Defaults: register windows (1), ring windows (0) for cfg5's column pass.  On the H100 the
// headline passes are HBM-bound and the variants are within noise of each other
// (profiles/h100_sweep.jsonl, L2 flushed between launches, same output hash for every variant:
// cfg3 row pass 0.329 / 0.329 / 0.330 ms for variants 0 / 1 / 3, column pass 0.166 / 0.168 /
// 0.170 / 0.169 ms for 0 / 1 / 2 / 3), so the defaults were kept.
inline int stream_default_variant(int chain, bool is_v) { return (is_v && chain == 5 /* kChainDil56 */) ? 0 : 1; }

struct StreamAxisPlan {
    int chain = kChainNone;
    int nsteps = 0;
    int src_len = 0, dst_len = 0;
    StreamStep s[kMaxSteps];
};

// What the compile-time chains expect of each step (mirrors the StepC arguments).
struct StepSpec {
    int kind, sum, nt, adv;
};

inline const StepSpec* chain_spec(int id, int* nsteps) {
    static const StepSpec dil24[] = {{K_RESIZE, AVIRB200_SUM_DIL8, 24, 2}, {K_FIR, AVIRB200_SUM_DIL8, 8, 1}};
    static const StepSpec inl24[] = {{K_RESIZE, AVIRB200_SUM_INL, 24, 2}, {K_FIR, AVIRB200_SUM_INL, 7, 1}};
    static const StepSpec inl3[] = {{K_FIR, AVIRB200_SUM_INL, 7, 1}, {K_RESIZE, AVIRB200_SUM_INL, 18, 2},
                                    {K_FIR, AVIRB200_SUM_INL, 7, 1}};
    static const StepSpec dil56[] = {{K_RESIZE, AVIRB200_SUM_DIL8, 56, 4}, {K_FIR, AVIRB200_SUM_DIL8, 8, 1}};
    static const StepSpec inl3d[] = {{K_FIR, AVIRB200_SUM_INL, 15, 2}, {K_RESIZE, AVIRB200_SUM_INL, 18, 2},
                                     {K_FIR, AVIRB200_SUM_INL, 7, 1}};
    static const StepSpec up2[] = {{K_FIR, AVIRB200_SUM_INL, 7, 1}, {K_RESIZE2, AVIRB200_SUM_INL, 24, 1}};
    switch (id) {
    case kChainDil24: case kChainDil24Q: *nsteps = 2; return dil24;
    case kChainInl24: *nsteps = 2; return inl24;
    case kChainInl3: *nsteps = 3; return inl3;
    case kChainInl3D: *nsteps = 3; return inl3d;
    case kChainDil56: *nsteps = 2; return dil56;
    case kChainUp2: *nsteps = 2; return up2;
    default: *nsteps = 0; return nullptr;
    }
}

// Fills `out` from one descriptor step if it has the shape `sp` asks for.
inline bool stream_match_step(const avirb200_step_desc& d, const StepSpec& sp, StreamStep& out) {
    memset(&out, 0, sizeof out);
    out.out_len = d.out_len;
    out.in_len = d.in_len;
    out.zero_start = d.zero_start;
    out.taps[kTapOne].lo = out.taps[kTapOne].hi = 1.0f;
    if (sp.kind == K_FIR) {
        if (d.kind != AVIRB200_STEP_FIR || d.ntaps != sp.nt || d.resample != sp.adv) return false;
        if (sp.sum == AVIRB200_SUM_INL && d.ntaps != 2 * d.latency + 1) return false;
        out.edge = d.edge;
        out.latency = d.latency;
        for (int t = 0; t < d.ntaps; ++t) out.taps[t].lo = out.taps[t].hi = d.taps[t];
        return true;
    }
    if (d.kind != AVIRB200_STEP_RESIZE || d.ntaps != sp.nt || d.ntaps > 64 || d.out_len < 1) return false;
    if (sp.kind == K_RESIZE && d.upsampled) return false;
    if (sp.kind == K_RESIZE2 && !(d.upsampled && d.skip_odd)) return false;
    const int step = (sp.kind == K_RESIZE2) ? 1 : sp.adv;
    uint32_t f0 = 0;
    if (d.order) memcpy(&f0, &d.frac[0], 4);
    for (int j = 0; j < d.out_len; ++j) {
        if (d.src_pos[j] != d.src_pos[0] + step * j) return false; // constant source step
        if (d.phase[j] != d.phase[0]) return false;                // one effective phase
        if (d.order) {
            uint32_t fj;
            memcpy(&fj, &d.frac[j], 4);
            if (fj != f0) return false;
        }
    }
    out.sp_first = d.src_pos[0];
    // effective taps c0 + c1*x: the two float operations upstream performs per tap
    // (avir.h:3945, avir_dil.h:649-650)
    const float* c0 = d.taps + (size_t)d.phase[0] * d.ntaps * (d.order + 1);
    for (int t = 0; t < d.ntaps; ++t) {
        if (d.order) {
            volatile float prod = c0[d.ntaps + t] * d.frac[0];
            out.taps[t].lo = c0[t] + prod;
        } else {
            out.taps[t].lo = c0[t];
        }
        out.taps[t].hi = out.taps[t].lo;
    }
    return true;
}

// Decides whether the axis runs on the streaming kernel; on success `out` holds everything
// the kernel parameters need.
inline bool stream_plan_axis(const avirb200_axis_desc& ad, int sum_mode, int channels, StreamAxisPlan& out,
                             int allow_deselected = 0, bool is_v = false) {
    out.chain = kChainNone;
    if (channels != 4) return false;
    // allow_deselected (AVIRB200_OPT_ALL_STREAM_CHAINS): the upsizing chain is instantiated and
    // checked for both passes but its COLUMN pass is not selected by default (the tile kernel's
    // blocked skip-odd resize is used there; not re-measured on the H100).
    for (int id = 1; id < kChainCount; ++id) {
        if (id == kChainUp2 && is_v && !allow_deselected) continue;
        if (id == kChainDil24Q && allow_deselected != 2) continue;
        if (id == kChainDil24 && allow_deselected == 2) continue;
        int ns = 0;
        const StepSpec* spec = chain_spec(id, &ns);
        if (ns != ad.nsteps) continue;
        bool ok = true;
        int prev = ad.src_len;
        for (int i = 0; i < ns && ok; ++i) {
            ok = (spec[i].sum == sum_mode) && ad.steps[i].in_len == prev &&
                 stream_match_step(ad.steps[i], spec[i], out.s[i]);
            prev = ad.steps[i].out_len;
        }
        if (!ok || prev != ad.dst_len) continue;
        out.chain = id;
        out.nsteps = ns;
        out.src_len = ad.src_len;
        out.dst_len = ad.dst_len;
        return true;
    }
    return false;
}

// The row pass streams the caller's pixels into shared memory as they are (cp.async); integer
// pixels are cast in the compute lanes' own reads.  Sources that need the sRGB linearisation
// on the way in stay on the tile kernel (it converts every sample once, in double) -- except
// u8, whose linearisation is a 256-entry table.
inline bool stream_row_source_ok(const avirb200_plan_desc& d) {
    if (d.use_gamma & 1) return d.in_type == AVIRB200_U8;
    return d.in_type == AVIRB200_F32 || d.in_type == AVIRB200_U8 || d.in_type == AVIRB200_U16;
}
// Output stage of the column pass, a compile-time choice of the kernel: 1 = float
// destination without output gamma (store as is), 2 = integer destination without output gamma
// and without bit-depth truncation (round, clamp, narrow; branch-free), 0 = everything (sRGB de-linearisation in double included -- its code
// is large enough to slow the whole kernel down, hence the split).
// 16-line strips of a launch (a segmented launch cuts each segment into strips of its own).
#if defined(__CUDACC__)
__host__ __device__
#endif
inline int stream_strip_count(const StreamParams& p) {
    if (p.seg_b > 0) return (p.seg_a + 15) / 16 + (p.seg_b + 15) / 16;
    return (p.n_lines + 15) / 16;
}
inline int stream_epilogue_code(const avirb200_plan_desc& d) {
    if (d.use_gamma & 2) return 0;
    if (d.out_type == AVIRB200_F32) return 1;
    return d.tr_mul == 1.0f ? 2 : 0; // (bit-depth truncation: the run-time stage)
}
inline int stream_row_source_code(const avirb200_plan_desc& d) {
    return (d.use_gamma & 1) ? kSrcU8Srgb : d.in_type;
}

// ---- fused halo exchange of sharded calls (StreamParams xs_* / xr_*) --------------------------------
// A band's mailbox as the kernels see it: the rows received from the band above and from the band below,
// the two flags (flags[0]: the rows from above are in, flags[1]: the rows from below) and the two
// counters the band's own row pass keeps as sender (count[0]: rows going up, count[1]: down).
struct StreamMailbox {
    float* from_up = nullptr;
    float* from_dn = nullptr;
    unsigned* flags = nullptr;
    unsigned long long* count = nullptr;
};

// One band of a sharded call and its neighbours (up / dn: null at the ends of the image), with the
// mailboxes of all three for the call's sequence number.  The band sends its first up->halo_down rows
// to the band above and its last dn->halo_up rows to the band below.
struct StreamLink {
    const avirb200_shard_info* me = nullptr;
    const avirb200_shard_info* up = nullptr;
    const avirb200_shard_info* dn = nullptr;
    StreamMailbox mine, above, below;
    unsigned seq = 0;
};
inline int stream_rows_up(const StreamLink& l) { return l.up ? l.up->halo_down : 0; }
inline int stream_rows_down(const StreamLink& l) { return l.dn ? l.dn->halo_up : 0; }

// The fused halves run only between neighbours that exchange rows in BOTH directions.  Slots alternate
// per call and are reused two calls later; what orders the reuse is that a band's call n+1 needs its
// neighbour's call-n+1 rows, which the neighbour sends after its call-n column pass.
inline bool stream_fused_rx_ok(const StreamLink& l) {
    return (l.up == nullptr || (stream_rows_up(l) > 0) == (l.me->halo_up > 0)) &&
           (l.dn == nullptr || (stream_rows_down(l) > 0) == (l.me->halo_down > 0));
}
// The fused sender counts per direction over whole 16-line strips: not for a band so short that one
// strip holds rows of both neighbours.
inline bool stream_fused_tx_ok(const StreamLink& l) {
    const int top = stream_rows_up(l), bot = stream_rows_down(l);
    return stream_fused_rx_ok(l) && !(top > 0 && bot > 0 && (top + kLines - 1) / kLines > (l.me->src_rows - bot) / kLines);
}

// Row pass as sender: the band's boundary rows also go into the neighbours' mailboxes.
inline void stream_set_sender(StreamParams& p, const StreamLink& l) {
    const int top = stream_rows_up(l), bot = stream_rows_down(l), rows = l.me->src_rows;
    p.xs_seq = l.seq;
    p.xs_count = l.mine.count;
    if (top > 0) {
        p.xs_up_dst = l.above.from_dn;
        p.xs_up_flag = &l.above.flags[1];
        p.xs_top = top;
        p.xs_units[0] = (unsigned long long)((top + kLines - 1) / kLines);
    }
    if (bot > 0) {
        p.xs_dn_dst = l.below.from_up;
        p.xs_dn_flag = &l.below.flags[0];
        p.xs_bot0 = rows - bot;
        p.xs_bot = bot;
        p.xs_units[1] = (unsigned long long)((rows + kLines - 1) / kLines - p.xs_bot0 / kLines);
    }
}

// Column pass as receiver: the neighbours' rows are read in place from the band's own mailbox.
inline void stream_set_receiver(StreamParams& p, const StreamLink& l) {
    p.xr_up_src = l.mine.from_up;
    p.xr_dn_src = l.mine.from_dn;
    p.xr_flags = l.mine.flags;
    p.xr_seq = l.seq;
    p.xr_own_lo = l.me->src_row0;
    p.xr_own_hi = l.me->src_row0 + l.me->src_rows;
}

// Kernel parameters of the pass `q` (its buffers as the kernel sees them) on the axis plan `ap`.
inline void stream_params(StreamParams& p, const StreamAxisPlan& ap, const avirb200_plan_desc& d,
                          const avb::PassRequest& q, const float* lut) {
    memset(&p, 0, sizeof p);
    for (int i = 0; i < ap.nsteps; ++i) p.s[i] = ap.s[i];
    p.n_lines = q.lines;
    if (q.seg_bot > 0) {
        p.seg_a = q.seg_top;
        p.seg_b = q.seg_bot;
        p.seg_b_line0 = q.lines - q.seg_bot;
    } else if (q.seg_top > 0) {
        p.n_lines = q.seg_top;
    }
    p.src_len = ap.src_len;
    p.out0 = q.out0;
    p.out1 = q.out1;
    p.src = q.src;
    p.src_type = q.is_v ? AVIRB200_F32 : stream_row_source_code(d);
    p.src_pitch = (long long)q.src_pitch;
    p.src_row_base = q.src_base;
    p.src_lo = q.src_lo;
    p.src_hi = q.src_hi;
    p.dst = q.dst;
    p.dst_pitch = (long long)q.dst_pitch;
    p.dst_type = q.dst_type;
    p.dst_row_base = q.dst_base;
    const avb::PixelStage px = avb::pixel_stage(d, lut);
    p.srgb_lut = px.srgb_lut;
    p.in_gamma_mult = px.in_gamma_mult;
    p.gamma_out = px.gamma_out;
    p.alpha_index = px.alpha_index;
    p.out_gamma_mult = px.out_gamma_mult;
    p.round_mode = px.round_mode;
    p.tr_mul = px.tr_mul;
    p.tr_mul_inv = px.tr_mul_inv;
    p.pk_out = px.pk_out;
    if (q.link != nullptr) {
        if (q.is_v) stream_set_receiver(p, *q.link);
        else stream_set_sender(p, *q.link);
    }
}

// The CPU emulation's entry points (tests/emul): a row pass of `rows` whole source lines (seg_top / seg_bot:
// only its first and last lines, one launch; cols: only the intermediate columns [out0, out1) from a buffer
// holding source columns [src_lo, src_hi)), and a column pass over d.dst_w intermediate columns.  Both are
// requests for stream_params.
struct StreamColumns {
    int out0, out1, src_lo, src_hi;
};
inline void stream_fill_row_params(StreamParams& p, const StreamAxisPlan& ap, const avirb200_plan_desc& d,
                                   const void* src, long long src_pitch, float* mid, long long mid_pitch, int rows,
                                   const float* lut, int seg_top = 0, int seg_bot = 0,
                                   const StreamColumns* cols = nullptr) {
    avb::PassRequest q = avb::row_request(d, src, (size_t)src_pitch, rows, mid, (size_t)mid_pitch);
    q.seg_top = seg_top;
    q.seg_bot = seg_bot;
    if (cols != nullptr) {
        q.out0 = q.dst_base = cols->out0;
        q.out1 = cols->out1;
        q.src_base = q.src_lo = cols->src_lo;
        q.src_hi = cols->src_hi;
    }
    stream_params(p, ap, d, q, lut);
}
inline void stream_fill_col_params(StreamParams& p, const StreamAxisPlan& ap, const avirb200_plan_desc& d,
                                   const float* mid, long long mid_pitch, int mid_lo, int mid_hi, void* dst,
                                   long long dst_pitch, int out0, int out1) {
    stream_params(p, ap, d,
                  avb::col_request(d, d.dst_w, mid, (size_t)mid_pitch, mid_lo, mid_hi, dst, (size_t)dst_pitch, out0, out1),
                  nullptr);
}

} // namespace avs
