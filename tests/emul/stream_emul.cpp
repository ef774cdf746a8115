// stream_emul.cpp -- TEST INFRASTRUCTURE: lockstep host emulation of the warp-streaming pass
// kernel (avir_b200/csrc/stream_kernel.cuh).
//
// The kernel source is compiled here for the host: a warp is 32 threads that meet at a
// pthread barrier wherever the device code executes __syncwarp(), cp.async becomes an
// immediate 16-byte copy, "shared memory" is a per-warp heap block.  The emulation exists so
// that the kernel's index logic (rings, software-pipeline delays, run splitting, edge
// batches, shard ranges) can be checked bit-for-bit against the oracle on a machine without
// a GPU (tests/test_stream_emul.py).  It is never linked into libavirb200.so and is not a
// CPU execution path of the product.
//
// Build: g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC (tests/emul/build.py).

#include <pthread.h>
#include <stdlib.h>

#include <thread>
#include <vector>

#include <atomic>

static thread_local pthread_barrier_t* g_bar = nullptr;
void avs_emul_syncwarp() { pthread_barrier_wait(g_bar); }
static std::atomic<long> g_oob(0);
namespace avs {
thread_local const unsigned char* avs_emul_src_lo = nullptr;
thread_local const unsigned char* avs_emul_src_hi = nullptr;
thread_local const unsigned char* avs_emul_alt_lo[2] = {nullptr, nullptr};
thread_local const unsigned char* avs_emul_alt_hi[2] = {nullptr, nullptr};
void avs_emul_count_oob() { ++g_oob; }
unsigned long long avs_emul_xs_add(unsigned long long* c, unsigned long long v) { // (one lane of one warp at a time)
    const unsigned long long old = *c;
    *c = old + v;
    return old;
}
} // namespace avs
static const unsigned char* g_lo = nullptr; // bounds of the pass's source buffer (copied into every lane thread)
static const unsigned char* g_hi = nullptr;
static const unsigned char* g_alt_lo[2] = {nullptr, nullptr};
static const unsigned char* g_alt_hi[2] = {nullptr, nullptr};

#include "host_util.h"
#include "stream_kernel.cuh"

using namespace avs;
using avb::elem_size;

namespace {

template <class C, bool IS_V, int EPI>
void emul_pass(const StreamParams& p, int nwarps) {
    const size_t sm_float2 = (size_t)(IS_V ? C::WARP_F2_V : C::WARP_F2_H);
    for (int gw = 0; gw < nwarps; ++gw) {
        std::vector<float2> sm(sm_float2);
        // poison: reads of never-written slots must not go unnoticed
        for (auto& v : sm) v = make_float2(__builtin_nanf(""), __builtin_nanf(""));
        pthread_barrier_t bar;
        pthread_barrier_init(&bar, nullptr, 32);
        std::vector<std::thread> th;
        for (int lane = 0; lane < 32; ++lane) {
            th.emplace_back([&, lane] {
                g_bar = &bar;
                avs_emul_src_lo = g_lo;
                avs_emul_src_hi = g_hi;
                for (int q = 0; q < 2; ++q) { avs_emul_alt_lo[q] = g_alt_lo[q]; avs_emul_alt_hi[q] = g_alt_hi[q]; }
                stream_warp_main<C, IS_V, EPI>(p, gw, nwarps, lane, sm.data(), p.srgb_lut);
            });
        }
        for (auto& t : th) t.join();
        pthread_barrier_destroy(&bar);
    }
}

template <bool IS_V>
bool emul_dispatch(int chain, int variant, const StreamParams& p, int nwarps, int epi) {
    return stream_dispatch(chain, IS_V, variant, p.src_type, [&](auto tag, auto pass) {
        using C = typename decltype(tag)::type;
        if constexpr (decltype(pass)::is_v != IS_V) {
            (void)p; // (the dispatcher instantiates the callback for both passes)
        } else if constexpr (IS_V) {
            if (epi == 1) emul_pass<C, true, 1>(p, nwarps);
            else if (epi == 2) emul_pass<C, true, 2>(p, nwarps);
            else emul_pass<C, true, 0>(p, nwarps);
        } else {
            if (p.xs_count != nullptr) emul_pass<C, false, kEpiXs>(p, nwarps);
            else emul_pass<C, false, 0>(p, nwarps);
        }
    });
}

} // namespace

extern "C" {

// 1 when both axes of the descriptor run on the streaming kernel (f32 source only).
int stream_emul_applicable(const avirb200_plan_desc* d) {
    StreamAxisPlan h, v;
    return stream_row_source_ok(*d) && stream_plan_axis(d->h, d->sum_mode, d->channels, h, 1) &&
           stream_plan_axis(d->v, d->sum_mode, d->channels, v, 1);
}

// Row pass with `warps_h` emulated warps, then the column pass in `bands` destination bands
// (as the sharded schedule runs it) with `warps_v` warps each.
// lut: the 256-entry u8 sRGB linearisation table (read for sRGB sources only).
// allow: 1 = every chain (as AVIRB200_OPT_ALL_STREAM_CHAINS = 1), 2 = the 4-output-batch twin of the
// headline chain where it applies.
// need: per band (need_row0, need_rows) of avirb200_shard_query_desc, or null.  With it every band's
// column pass gets a buffer holding exactly those intermediate rows, as a rank of the sharded
// schedule does, and every source read is bounds-checked: returns -5 if any read left its buffer.
int stream_emul_resize(const avirb200_plan_desc* d, const void* src, size_t src_pitch, void* dst,
                       size_t dst_pitch, int warps_h, int warps_v, int bands, int variant, const float* lut, int allow,
                       const int* need, int seg_top, int seg_bot) {
    StreamAxisPlan h, v;
    if (!stream_row_source_ok(*d) || !stream_plan_axis(d->h, d->sum_mode, d->channels, h, allow) ||
        !stream_plan_axis(d->v, d->sum_mode, d->channels, v, allow))
        return -4;
    const size_t rowf = (size_t)d->dst_w * 4, in_es = elem_size(d->in_type), out_es = elem_size(d->out_type);
    std::vector<float> mid((size_t)d->src_h * rowf);
    StreamParams p;
    g_oob = 0;
    g_lo = static_cast<const unsigned char*>(src);
    g_hi = g_lo + ((size_t)(d->src_h - 1) * src_pitch + (size_t)d->src_w * 4) * in_es;
    if (seg_top + seg_bot > 0 && seg_top + seg_bot < d->src_h) {
        // as a sharded call schedules the row pass: the first seg_top and last seg_bot rows in one
        // segmented launch, then the rows between
        stream_fill_row_params(p, h, *d, src, (long long)src_pitch, mid.data(), (long long)rowf, d->src_h, lut, seg_top,
                               seg_bot);
        if (!emul_dispatch<false>(h.chain, variant, p, warps_h, 0)) return -4;
        stream_fill_row_params(p, h, *d, static_cast<const unsigned char*>(src) + (size_t)seg_top * src_pitch * in_es,
                               (long long)src_pitch, mid.data() + (size_t)seg_top * rowf, (long long)rowf,
                               d->src_h - seg_top - seg_bot, lut);
        if (!emul_dispatch<false>(h.chain, variant, p, warps_h, 0)) return -4;
    } else {
        stream_fill_row_params(p, h, *d, src, (long long)src_pitch, mid.data(), (long long)rowf, d->src_h, lut);
        if (!emul_dispatch<false>(h.chain, variant, p, warps_h, 0)) return -4;
    }

    const int epi = stream_epilogue_code(*d);
    for (int b = 0; b < bands; ++b) {
        const int out0 = (int)((long long)d->dst_h * b / bands), out1 = (int)((long long)d->dst_h * (b + 1) / bands);
        if (out1 <= out0) continue;
        const float* msrc = mid.data();
        int lo = 0, hi = d->src_h;
        std::vector<float> bandbuf;
        if (need != nullptr) { // the band's own rows only, as on a rank of the sharded schedule
            lo = need[2 * b];
            hi = lo + need[2 * b + 1];
            bandbuf.assign(mid.begin() + (size_t)lo * rowf, mid.begin() + (size_t)hi * rowf);
            msrc = bandbuf.data();
        }
        g_lo = reinterpret_cast<const unsigned char*>(msrc);
        g_hi = g_lo + (size_t)(hi - lo) * rowf * sizeof(float);
        stream_fill_col_params(p, v, *d, msrc, (long long)rowf, lo, hi,
                               static_cast<unsigned char*>(dst) + (size_t)out0 * dst_pitch * out_es, (long long)dst_pitch,
                               out0, out1);
        if (!emul_dispatch<true>(v.chain, variant, p, warps_v, epi)) return -4;
    }
    g_lo = g_hi = nullptr;
    return g_oob.load() ? -5 : 0;
}

// The sharded schedule with the FUSED halo exchange (AVIRB200_OPT_OVERLAP_HALO = 3): every band's row
// pass writes its own rows into its own buffer and the rows its neighbours need into their mailboxes
// (counting completed boundary rounds, then raising the neighbour's flag); every band's column pass
// reads its own rows from its buffer and the neighbours' rows in place from its mailbox.
// info: avirb200_shard_info of every band (8 ints each).  Every buffer is NaN-poisoned and exactly as
// large as the rows it is meant to hold; reads are bounds-checked (-5), flags and counters are
// checked after the row passes (-6).  The parameters and the eligibility rule are the engine's own
// (stream_types.h: stream_set_sender / _receiver, stream_fused_tx_ok).  Returns 1, nothing computed,
// where the product would not run the fused sender for some band.
int stream_emul_resize_fused(const avirb200_plan_desc* d, const void* src, size_t src_pitch, void* dst,
                             size_t dst_pitch, int warps_h, int warps_v, int bands, int variant, const float* lut,
                             int allow, const int* info) {
    StreamAxisPlan h, v;
    if (!stream_row_source_ok(*d) || !stream_plan_axis(d->h, d->sum_mode, d->channels, h, allow) ||
        !stream_plan_axis(d->v, d->sum_mode, d->channels, v, allow))
        return -4;
    struct Band {
        avirb200_shard_info si;
        std::vector<float> own, box_up, box_dn; // box_up: rows from the band above, box_dn: from the band below
        unsigned flags[2] = {0, 0};
        unsigned long long count[2] = {0, 0};
        StreamLink link;
    };
    const size_t rowf = (size_t)d->dst_w * 4, in_es = elem_size(d->in_type), out_es = elem_size(d->out_type);
    const float nanv = __builtin_nanf("");
    const unsigned seq = 5;
    std::vector<Band> B(bands);
    for (int b = 0; b < bands; ++b) {
        Band& x = B[b];
        memcpy(&x.si, info + 8 * b, sizeof x.si);
        x.own.assign((size_t)x.si.src_rows * rowf, nanv);
        x.box_up.assign((size_t)x.si.halo_up * rowf, nanv);
        x.box_dn.assign((size_t)x.si.halo_down * rowf, nanv);
        x.link.me = &x.si;
        x.link.mine = {x.box_up.data(), x.box_dn.data(), x.flags, x.count};
        x.link.seq = seq;
    }
    for (int b = 0; b < bands; ++b) {
        StreamLink& l = B[b].link;
        if (b > 0) { l.up = &B[b - 1].si; l.above = B[b - 1].link.mine; }
        if (b + 1 < bands) { l.dn = &B[b + 1].si; l.below = B[b + 1].link.mine; }
        if (stream_rows_up(l) > B[b].si.src_rows || stream_rows_down(l) > B[b].si.src_rows) return -4;
        if (!stream_fused_tx_ok(l)) return 1; // the product runs the copy-engine exchange
    }
    g_oob = 0;
    g_alt_lo[0] = g_alt_lo[1] = g_alt_hi[0] = g_alt_hi[1] = nullptr;
    StreamParams p;
    for (int b = 0; b < bands; ++b) {
        Band& x = B[b];
        const unsigned char* bsrc = static_cast<const unsigned char*>(src) + (size_t)x.si.src_row0 * src_pitch * in_es;
        stream_fill_row_params(p, h, *d, bsrc, (long long)src_pitch, x.own.data(), (long long)rowf, x.si.src_rows, lut);
        stream_set_sender(p, x.link);
        g_lo = bsrc;
        g_hi = g_lo + ((size_t)(x.si.src_rows - 1) * src_pitch + (size_t)d->src_w * 4) * in_es;
        if (!emul_dispatch<false>(h.chain, variant, p, warps_h, 0)) return -4;
        if (x.count[0] != 0 || x.count[1] != 0) return -6;
        if (stream_rows_up(x.link) > 0 && B[b - 1].flags[1] != seq) return -6;
        if (stream_rows_down(x.link) > 0 && B[b + 1].flags[0] != seq) return -6;
    }
    const int epi = stream_epilogue_code(*d);
    for (int b = 0; b < bands; ++b) {
        Band& x = B[b];
        if (x.si.dst_rows <= 0) continue;
        // (row need_row0 of a buffer that only holds the own rows)
        stream_fill_col_params(p, v, *d, x.own.data() - (ptrdiff_t)x.si.halo_up * (ptrdiff_t)rowf, (long long)rowf,
                               x.si.need_row0, x.si.need_row0 + x.si.need_rows,
                               static_cast<unsigned char*>(dst) + (size_t)x.si.dst_row0 * dst_pitch * out_es,
                               (long long)dst_pitch, x.si.dst_row0, x.si.dst_row0 + x.si.dst_rows);
        stream_set_receiver(p, x.link);
        g_lo = reinterpret_cast<const unsigned char*>(x.own.data());
        g_hi = g_lo + x.own.size() * sizeof(float);
        g_alt_lo[0] = reinterpret_cast<const unsigned char*>(x.box_up.data());
        g_alt_hi[0] = g_alt_lo[0] + x.box_up.size() * sizeof(float);
        g_alt_lo[1] = reinterpret_cast<const unsigned char*>(x.box_dn.data());
        g_alt_hi[1] = g_alt_lo[1] + x.box_dn.size() * sizeof(float);
        if (x.box_up.empty()) g_alt_lo[0] = g_alt_hi[0] = nullptr;
        if (x.box_dn.empty()) g_alt_lo[1] = g_alt_hi[1] = nullptr;
        if (!emul_dispatch<true>(v.chain, variant, p, warps_v, epi)) return -4;
    }
    g_lo = g_hi = nullptr;
    g_alt_lo[0] = g_alt_lo[1] = g_alt_hi[0] = g_alt_hi[1] = nullptr;
    return g_oob.load() ? -5 : 0;
}

int stream_emul_variants(void) { return kStreamVariants; }

// What the engine would choose for the descriptor: out[0] / out[1] = StreamChainId of the row /
// column pass (0 = the pass runs on the tile or generic kernel), out[2] = row-pass source code,
// out[3] = column-pass epilogue code.  all_chains: as with AVIRB200_STREAM_ALL=1.
void stream_emul_selection(const avirb200_plan_desc* d, int all_chains, int* out) {
    StreamAxisPlan h, v;
    out[0] = (stream_row_source_ok(*d) && stream_plan_axis(d->h, d->sum_mode, d->channels, h, all_chains, false))
                 ? h.chain : 0;
    out[1] = stream_plan_axis(d->v, d->sum_mode, d->channels, v, all_chains, true) ? v.chain : 0;
    out[2] = stream_row_source_code(*d);
    out[3] = stream_epilogue_code(*d);
}

} // extern "C"
