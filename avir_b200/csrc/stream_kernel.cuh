// stream_kernel.cuh -- warp-streaming pass kernel for regular 4-channel chains (sm_90a).
//
// The tile kernel (fast_kernel.cuh) gives every block a tile of 16 lines, runs one step of
// the chain at a time over the whole tile and separates the steps with block barriers.  With
// the shared memory a chain needs, a tile holds ~130 outputs, i.e. 2-3 inner-loop trips per
// warp between barriers: the FP32 pipe idles half of the time.  This kernel removes the
// barriers altogether:
//
//   * a WARP owns a run: 16 lines (lane = one channel pair of one line, as in the tile
//     kernel) times a long contiguous range of positions, and streams along it;
//   * every step of the chain works in batches of 8 outputs from a register window of its
//     input (38 shared loads per 376 packed FP instructions for the 24-tap resize) and appends the
//     batch to a small per-warp ring in shared memory; the next step consumes that ring a
//     fixed number of rounds later (software pipeline, all offsets compile-time);
//   * a lane only ever reads back what it wrote itself ([position][lane] layout), so the
//     intermediate rings need no synchronisation at all; only the source ring (filled by
//     cp.async copies of whole pixels -- float, or the caller's u8 / u16 pixels as they are,
//     cast in the lanes' reads -- up to three rounds ahead of use) and the row pass's output
//     staging use __syncwarp;
//   * taps are kernel parameters (uniform-register operands of the packed multiplies, see
//     f2mul / f2add below): only chains
//     whose resize step has one effective phase and a constant source step -- all integer
//     ratios, i.e. every BASELINE configuration -- run here, everything else stays on the
//     tile kernel;
//   * edges: the source ring materialises the replicated border (the loader clamps the
//     global coordinate); a batch whose window leaves its input line, or that is cut by the
//     end of its own output line, takes a per-output path that clamps every tap position
//     (upstream replicates edges per step, avir.h:3227-3239) -- 2 batches per line and step.
//
// Arithmetic (order of the separate multiplies and adds) is the tile kernel's, i.e.
// upstream's; tests compare all three kernels against the oracle.  The same source compiles
// for the host (tests/emul/stream_emul.cpp: 32 threads in lockstep per warp) so that the
// index logic is checked against the oracle on machines without a GPU.
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "avirb200.h"
#include "pixel_ops.cuh"
#include "stream_types.h"

#if defined(__CUDACC__)
#define AVS_FN __device__ __forceinline__
#define AVS_SYNCWARP() __syncwarp()
#else
#define AVS_FN inline __attribute__((always_inline))
void avs_emul_syncwarp(); // the emulator's lockstep barrier
#define AVS_SYNCWARP() avs_emul_syncwarp()
#endif

namespace avs {

using avb::lin2srgb;
using avb::round_out;
using avb::round_out_int;

constexpr int kEpiXs = 4;       // row pass "epilogue" code: sender of the fused halo exchange (StreamParams xs_*)
constexpr int kPitchL = 32;     // float2 units: [position][lane] rows of 256 bytes
// Row pass, source ring and output staging: [line][position][4 channels] with one pixel of
// padding per line.  The copies into it (cp.async) and out of the staging rows then move
// runs of whole pixels of a row -- 256 contiguous bytes per half warp on both sides -- and
// the transposition into lanes (lane = line x channel pair) happens in the compute lanes'
// own 8-byte reads and writes, which the padding keeps conflict-free (16 lines fall into 8
// distinct 16-byte bank groups twice: two wavefronts, the minimum for 256 bytes).

// Compile-time description of one step.  NT = taps (FIR: stored taps, 2L+1 for the
// interleaved form, padded to 8 for the de-interleaved one; RESIZE/RESIZE2: filter length).
// ADV = input positions per output (FIR decimation R, RESIZE source step D).
// RESIZE2 = resize over the virtual 2X zero-stuffed line, odd taps skipped (upstream
// doResize2, avir.h:4114-4328): two outputs per input position.
// MB = outputs per batch (0: 8, or 16 for RESIZE2; 4 for the long cfg5 filter: its window would
// not fit the register file otherwise).
template <int KIND_, int SUM_, int NT_, int ADV_, int MB_ = 0>
struct StepC {
    static constexpr int KIND = KIND_, SUM = SUM_, NT = NT_, ADV = ADV_;
    static constexpr int M = (KIND == K_RESIZE2) ? 16 : (MB_ ? MB_ : 8); // outputs per batch
    static constexpr int CH = (KIND == K_RESIZE2) ? 8 : M * ADV;    // input positions per batch
    static constexpr int NTW = (KIND == K_RESIZE2) ? NT / 2 : NT;   // inputs one output reads
    static constexpr int W = (KIND == K_RESIZE2) ? 20 : NT + (M - 1) * ADV; // window of a batch
};
using NoStep = StepC<K_NONE, 0, 0, 1>;

constexpr int cdiv(int a, int b) { return (a + b - 1) / b; }

// Compile-time software-pipeline schedule of a chain (see run_warp()).
//   reps[i]  batches of step i per round
//   delay[i] rounds step i lags behind step 0
//   rsp[i]   positions in the ring step i reads (ring 0 = source)
//   SRCT     element type of the row pass's source image (AVIRB200_F32 / _U8 / _U16): integer
//            pixels stream into the source ring as they are (4 / 8 bytes per pixel) and are
//            converted -- upstream's packScanline cast, avir.h:2777-2971 -- in the lanes' reads
//   MODE     scheduling of the interior ("steady") rounds of a run, same arithmetic:
//            0 ring windows (every batch reads its whole window from the shared-memory rings),
//            1 register windows (run_regwin(): every input is read from shared memory once and
//              slides through a register window; later steps never touch shared memory),
//            2 = 1 + mbarrier-tracked source ring filled by one-lane tensor copies (TMA; column pass),
//            3 = 0 without the separate straight-line loop (every round takes the checked path)
//   NWMAX    warps per block the chain aims for (8: two per scheduler; 12 where registers -- at most
//            168 a thread -- and the per-warp rings allow three)
template <class S0, class S1, class S2, int REPS_LAST, int LA, int MODE_ = 0, int SRCT_ = AVIRB200_F32, int RWU_ = 1,
          int NWMAX_ = 8>
struct ChainC {
    using T0 = S0;
    using T1 = S1;
    using T2 = S2;
    static constexpr int SRCT = SRCT_;
    static constexpr int PIXB = (SRCT == AVIRB200_F32) ? 16 : (SRCT == AVIRB200_U16 ? 8 : 4); // bytes per source pixel (u8, u8 sRGB: 4)
    static constexpr int NS = (S2::KIND == K_NONE) ? 2 : 3;
    static constexpr int LOOKAHEAD = LA;
    static constexpr int MODE = MODE_;
    static constexpr bool STEADY_LOOP = (MODE_ != 3); // straight-line code for the interior rounds of a run
    static constexpr bool REGWIN = (MODE_ == 1 || MODE_ == 2) && S0::KIND != K_RESIZE2 && S1::KIND != K_RESIZE2 &&
                                   S2::KIND != K_RESIZE2;
    // source ring filled by one-lane tensor copies (TMA) and tracked by mbarriers instead of
    // per-lane cp.async groups: column pass only (ChainV maps the row pass's mode 2 to mode 1 --
    // its ring is [line][position] with padded lines, which no dense TMA box lands as)
    static constexpr bool MBAR = (MODE_ == 2) && REGWIN;
    // register-window rounds per trip of the unrolled loop (run_regwin())
    static constexpr int RW_UNROLL = RWU_;
    static constexpr int reps2 = (NS == 3) ? REPS_LAST : 0;
    static constexpr int reps1 = (NS == 3) ? (S2::CH * reps2) / S1::M : REPS_LAST;
    static constexpr int reps0 = (S1::CH * reps1) / S0::M;
    static_assert(NS == 2 || (S2::CH * reps2) % S1::M == 0, "step 1 batches per round");
    static_assert((S1::CH * reps1) % S0::M == 0, "step 0 batches per round");
    static constexpr int B = (NS == 3) ? S2::M * reps2 : S1::M * reps1; // final outputs per round
    static constexpr int SRC_N = S0::CH * reps0;                        // source positions per round
    // the loader moves a group in sweeps of POSW positions x 16 lines, NK copies per lane
    static constexpr int POSW = (SRC_N >= 16) ? 16 : SRC_N;
    static constexpr int NK = POSW / 2;
    static_assert(SRC_N % POSW == 0 && (POSW == 16 || POSW == 8), "source positions per round: whole 8- or 16-position sweeps");
    // consumer i+1 needs its producer d rounds ahead
    static constexpr int d0 = cdiv(cdiv(S1::W, S1::CH) - 1, reps1);
    static constexpr int d1 = (NS == 3) ? cdiv(cdiv(S2::W, S2::CH) - 1, reps2) : 0;
    static constexpr int delay0 = 0, delay1 = d0, delay2 = d0 + d1;
    static constexpr int DELAY_LAST = (NS == 3) ? delay2 : delay1;
    static constexpr int rsp1 = S1::CH * reps1 * (d0 + 1);
    static constexpr int rsp2 = (NS == 3) ? S2::CH * reps2 * (d1 + 1) : 0;
    // source ring: groups of SRC_N positions; step 0's window overhangs h groups
    static constexpr int H = cdiv(S0::W - S0::CH, SRC_N);
    static constexpr int NG = H + LA + 1;
    static constexpr int rsp0 = NG * SRC_N;
    static constexpr int MLAST = (NS == 3) ? S2::M : S1::M;

    // shared memory of one warp, in float2 units
    static constexpr int LINE_B = (rsp0 + 1) * PIXB; // row pass: bytes per line of the source ring (one pixel of padding)
    static constexpr int SRC_RING_F2 = (kLines * LINE_B + 15) / 16 * 2;
    static constexpr int STAGE_LINE = MLAST * 2 + 2;
    // one 8-byte mbarrier per source-ring group; padded so that every warp's block (and with it
    // its source ring, the destination of the tensor copies) stays 128-byte aligned
    static constexpr int MBAR_F2 = MBAR ? 16 * ((NG + 15) / 16) : 0;
    static_assert(!MBAR || ((rsp0 * kPitchL + (rsp1 + rsp2) * kPitchL) % 16 == 0), "ring rows are 256 bytes");
    static constexpr int WARP_F2_H = SRC_RING_F2 + (rsp1 + rsp2) * kPitchL + kLines * STAGE_LINE + MBAR_F2;
    static constexpr int WARP_F2_V = rsp0 * kPitchL + (rsp1 + rsp2) * kPitchL + MBAR_F2;
    // warps per block (one block per SM): 8 (two per scheduler; the register windows leave room
    // for no more), fewer where the rings of 8 warps exceed the shared memory of an SM
    static constexpr int kSmemF2 = 227 * 1024 / 8;
    static constexpr int NWARPS_H = (NWMAX_ * WARP_F2_H <= kSmemF2) ? NWMAX_ : kSmemF2 / WARP_F2_H;
    static constexpr int NWARPS_V = (NWMAX_ * WARP_F2_V <= kSmemF2) ? NWMAX_ : kSmemF2 / WARP_F2_V;
    static_assert(NWARPS_H >= 4 && NWARPS_V >= 4, "per-warp rings too large");
};

// ---- small helpers ---------------------------------------------------------------------------------

AVS_FN int imin_(int a, int b) { return a < b ? a : b; }
AVS_FN int imax_(int a, int b) { return a > b ? a : b; }

// The two channels a lane owns travel as one pair.  Upstream multiplies and adds separately
// (two roundings per tap), so every product and sum is its own IEEE FMUL / FADD: sm_90 has no
// packed FP32 instructions, and __fmul_rn / __fadd_rn are never contracted into an FFMA.
AVS_FN float2 f2mul(const StreamTap& t, float2 x) { return make_float2(__fmul_rn(t.lo, x.x), __fmul_rn(t.hi, x.y)); }
AVS_FN float2 f2add(float2 a, float2 b, const StreamTap&) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
AVS_FN float2 f2hadd8(const float2* v, const StreamTap& one) {
    // float8::hadd (avir_float8_avx.h:264-273)
    return f2add(f2add(f2add(v[0], v[4], one), f2add(v[1], v[5], one), one),
                 f2add(f2add(v[2], v[6], one), f2add(v[3], v[7], one), one), one);
}

#if defined(__CUDACC__)
AVS_FN void cp_async16(void* smem, const void* gmem) {
    const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(gmem) : "memory");
}
// N bytes (4, 8: one integer pixel; through L1, the only form the small sizes have)
template <int N>
AVS_FN void cp_async_px(void* smem, const void* gmem) {
    if (N == 16) {
        cp_async16(smem, gmem);
    } else {
        const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
        asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(sa), "l"(gmem), "n"(N) : "memory");
    }
}
AVS_FN void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
AVS_FN void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// ---- mbarrier-tracked staging (C::MBAR): one barrier per source-ring group, 32 arrivals per phase
AVS_FN unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
AVS_FN void mbar_init(unsigned bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
AVS_FN void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
AVS_FN void mbar_arrive(unsigned bar) {
    asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.shared::cta.b64 st, [%0];\n}" ::"r"(bar) : "memory");
}
AVS_FN void mbar_arrive_expect_tx(unsigned bar, unsigned bytes) {
    asm volatile("{\n.reg .b64 st;\nmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n}" ::"r"(bar), "r"(bytes) : "memory");
}
// the lane's arrival fires when all cp.async copies it has issued so far have landed
AVS_FN void mbar_arrive_cp_async(unsigned bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(bar) : "memory");
}
// Bounded wait: a protocol error traps instead of hanging the device.
AVS_FN void mbar_wait(unsigned bar, unsigned parity) {
    unsigned done = 0;
#pragma unroll 1
    for (int spin = 0; spin < (1 << 24); ++spin) {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) return;
    }
    __trap();
}
// one 2-D tile (TMA): box of the tensor map at element coordinates (c0, c1) -> shared memory,
// completion counted in bytes on `bar`
AVS_FN void tma_tile_2d(void* dst, const void* tmap, int c0, int c1, unsigned bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(bar) : "memory");
}
#else
// host emulation: copies are immediate, barriers have nothing to wait for
AVS_FN unsigned smem_u32(const void*) { return 0; }
AVS_FN void mbar_arrive(unsigned) {}
AVS_FN void mbar_arrive_expect_tx(unsigned, unsigned) {}
AVS_FN void mbar_arrive_cp_async(unsigned) {}
AVS_FN void mbar_wait(unsigned, unsigned) {}
// (every source read of the emulation is checked against the buffer the pass was given)
extern thread_local const unsigned char* avs_emul_src_lo;
extern thread_local const unsigned char* avs_emul_src_hi;
extern thread_local const unsigned char* avs_emul_alt_lo[2]; // (fused halo exchange: the two mailbox areas)
extern thread_local const unsigned char* avs_emul_alt_hi[2];
void avs_emul_count_oob();
AVS_FN void emul_copy(void* smem, const void* gmem, int n) {
    const unsigned char* g = static_cast<const unsigned char*>(gmem);
    const bool in_alt = (avs_emul_alt_lo[0] != nullptr && g >= avs_emul_alt_lo[0] && g + n <= avs_emul_alt_hi[0]) ||
                        (avs_emul_alt_lo[1] != nullptr && g >= avs_emul_alt_lo[1] && g + n <= avs_emul_alt_hi[1]);
    if (avs_emul_src_lo != nullptr && !in_alt && (g < avs_emul_src_lo || g + n > avs_emul_src_hi)) {
        avs_emul_count_oob();
        memset(smem, 0xff, n);
        return;
    }
    memcpy(smem, gmem, n);
}
AVS_FN void cp_async16(void* smem, const void* gmem) { emul_copy(smem, gmem, 16); }
template <int N>
AVS_FN void cp_async_px(void* smem, const void* gmem) { emul_copy(smem, gmem, N); }
AVS_FN void cp_async_commit() {}
template <int N>
AVS_FN void cp_async_wait() {}
#endif

// ---- fused halo exchange: counters and flags ------------------------------------------------------------------
#if defined(__CUDACC__)
AVS_FN unsigned long long xs_add(unsigned long long* c, unsigned long long v) { return atomicAdd(c, v); }
AVS_FN void xs_publish(unsigned* flag, unsigned seq) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(seq) : "memory");
}
AVS_FN void xs_fence() { __threadfence_system(); }
AVS_FN void xr_wait(const volatile unsigned* flag, unsigned seq) {
    long long spins = 0;
    while ((int)(*flag - seq) < 0) {
        if (++spins > (1ll << 30)) __trap(); // the neighbour never delivered: fail instead of hanging
        __nanosleep(64);
    }
    __threadfence_system();
}
#else
unsigned long long avs_emul_xs_add(unsigned long long* c, unsigned long long v); // (atomic in the emulator)
AVS_FN unsigned long long xs_add(unsigned long long* c, unsigned long long v) { return avs_emul_xs_add(c, v); }
AVS_FN void xs_publish(unsigned* flag, unsigned seq) { *flag = seq; }
AVS_FN void xs_fence() {}
AVS_FN void xr_wait(const volatile unsigned* flag, unsigned seq) { // (bands run one after another: must be there)
    if ((int)(*flag - seq) < 0) avs_emul_count_oob();
}
#endif

// First input position output j of a step reads.
template <class S>
AVS_FN int in_first(const StreamStep& sp, int j) {
    if (S::KIND == K_FIR) return (j - sp.edge) * S::ADV - sp.latency;
    if (S::KIND == K_RESIZE) return sp.sp_first + S::ADV * j - (S::NT / 2 - 1);
    const int pv = sp.sp_first + j - (S::NT / 2 - 1); // virtual (2X) position
    return (pv + (pv & 1)) >> 1;
}

// ---- arithmetic of one output from a register window (x[off ...]) ------------------------------

template <class S, class X>
AVS_FN float2 fir_one(const X& x, const int off, const StreamTap* t) {
    const StreamTap& one = t[kTapOne];
    if (S::SUM == AVIRB200_SUM_DIL8) {
        float2 ln[8];
#pragma unroll
        for (int g = 0; g < S::NT / 8; ++g) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float2 v = f2mul(t[g * 8 + q], x[off + g * 8 + q]);
                ln[q] = (g == 0) ? v : f2add(ln[q], v, one);
            }
        }
        return f2hadd8(ln, one);
    }
    constexpr int L = S::NT / 2;
    float2 s = f2mul(t[L], x[off + L]);
#pragma unroll
    for (int i = 1; i <= L; ++i) s = f2add(s, f2mul(t[L + i], f2add(x[off + L + i], x[off + L - i], one)), one);
    return s;
}

template <class S, class X>
AVS_FN float2 resize_one(const X& x, const int off, const StreamTap* t, int zero_start) {
    const StreamTap& one = t[kTapOne];
    float2 r;
    if (S::SUM == AVIRB200_SUM_DIL8) {
        float2 ln[8];
#pragma unroll
        for (int g = 0; g < S::NT / 8; ++g) {
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float2 v = f2mul(t[g * 8 + q], x[off + g * 8 + q]);
                ln[q] = (g == 0) ? v : f2add(ln[q], v, one);
            }
        }
        r = f2hadd8(ln, one);
    } else {
        r = f2mul(t[0], x[off]);
#pragma unroll
        for (int i = 1; i < S::NT; ++i) r = f2add(r, f2mul(t[i], x[off + i]), one);
    }
    if (zero_start) r = f2add(r, make_float2(0.0f, 0.0f), one);
    return r;
}

// fo = parity of the output's first virtual position = index of its first tap
template <class S, class X>
AVS_FN float2 resize2_one(const X& x, const int off, const int fo, const StreamTap* t, int zero_start) {
    const StreamTap& one = t[kTapOne];
    float2 r = f2mul(t[fo], x[off]);
#pragma unroll
    for (int k = 1; k < S::NT / 2; ++k) r = f2add(r, f2mul(t[fo + 2 * k], x[off + k]), one);
    if (zero_start) r = f2add(r, make_float2(0.0f, 0.0f), one);
    return r;
}

// ---- output stage ---------------------------------------------------------------------------------------

// integer destinations: round (the class's own round()), clamp (avir.h:4392-4419)
AVS_FN float epilogue_round(const StreamParams& p, float v) {
    if (p.tr_mul == 1.0f) v = round_out(v, p.round_mode);
    else v = __fmul_rn(round_out(__fmul_rn(v, p.tr_mul_inv), p.round_mode), p.tr_mul);
    return v < 0.0f ? 0.0f : (v > p.pk_out ? p.pk_out : v);
}

// gamma_done: the output gamma has been applied to v already (epilogue_gamma_batch)
AVS_FN float epilogue_value(const StreamParams& p, float v, int c, bool gamma_done = false) {
    if (p.gamma_out && !gamma_done) {
        if (c == p.alpha_index) v = __fmul_rn(v, p.out_gamma_mult);
        else v = __fmul_rn(lin2srgb(v), p.out_gamma_mult);
    }
    if (p.dst_type != AVIRB200_F32) v = epilogue_round(p, v);
    return v;
}

// The output gamma of a lane's whole batch (M outputs x 2 channels, first channel c0) at once: the
// samples' square-root chains advance together (pixel_ops.cuh, lin2srgb_batch) instead of one after
// another.  Returns false, o untouched, when a sample needs the one-sample path (NaN, infinity).
template <int M>
AVS_FN bool epilogue_gamma_batch(const StreamParams& p, float2 (&o)[M], int c0) {
    float v[2 * M];
    bool ok = true;
#pragma unroll
    for (int m = 0; m < M; ++m) {
        v[2 * m] = o[m].x;
        v[2 * m + 1] = o[m].y;
        ok = ok && avb::lin2srgb_batch_ok(o[m].x) && avb::lin2srgb_batch_ok(o[m].y);
    }
    if (!ok) return false;
    // (at most 8 chains in flight: 16 would not fit the registers beside the windows)
    constexpr int G = (2 * M > 8) ? 8 : 2 * M;
#pragma unroll
    for (int i = 0; i < 2 * M; i += G) avb::lin2srgb_batch<G>(v + i);
    const bool a0 = (c0 == p.alpha_index), a1 = (c0 + 1 == p.alpha_index); // the alpha channel is exempt
#pragma unroll
    for (int m = 0; m < M; ++m) {
        o[m].x = __fmul_rn(avb::fsel(a0, o[m].x, v[2 * m]), p.out_gamma_mult);
        o[m].y = __fmul_rn(avb::fsel(a1, o[m].y, v[2 * m + 1]), p.out_gamma_mult);
    }
    return true;
}

// ---- per-warp state of a run -------------------------------------------------------------------------

struct SrcConv {
    const float* lut;
    float gm;
    bool alpha0, alpha1;
};

template <class C, bool IS_V>
struct WarpRun {
    float2* ring0;  // source ring
    float2* ring1;
    float2* ring2;
    float2* stage;  // row pass: transposition buffer of the final batch
    int lane, line0, nlines;
    SrcConv cv;     // row pass, sRGB source
    int o0;         // source position held by slot 0 of ring 0
    int a[kMaxSteps];   // output index of batch 0 of every step (= origin of the next ring)
    int rd[kMaxSteps];  // read slot (positions) of each step in its input ring
    int wr[kMaxSteps];  // write slot of each step in its output ring
    int kb[kMaxSteps];  // batches done
    // loader: one global pointer per cp.async of a sweep, advancing by 16 positions per sweep
    // (they point one sweep behind and are advanced BEFORE use: the copies read them in place
    // and the next write to them is a whole round away -- no write-after-read wait on the
    // copy queue)
    const unsigned char* gp[C::MBAR ? 1 : C::NK];
    // row pass: the previous final batch, read back from the staging rows, waiting to be stored
    float4 pend[C::MLAST / 2];
    int pend_j0;
    // source ring tracked by mbarriers (C::MBAR): shared address of slot 0's barrier, the phase
    // parity each slot's next completion will have (bit s = slot s)
    unsigned mbar0, mpar;
    // row pass of a sharded band, fused halo exchange: lines [xs_l0, xs_l1) of this run's strip are rows a
    // neighbour rank needs (xs_dir: 0 the rank above, 1 below); their copies live xs_delta bytes away
    int xs_l0, xs_l1, xs_dir;
    ptrdiff_t xs_delta;
};

template <class C, bool IS_V, int I>
struct RingOf {
    static constexpr int RSP = (I == 0) ? C::rsp0 : (I == 1 ? C::rsp1 : C::rsp2);
    // the row pass's source ring holds raw pixels [line][position]; every other ring float2 [position][lane]
    static constexpr bool RAW = (I == 0 && !IS_V);
    static constexpr int SRCT = RAW ? C::SRCT : AVIRB200_F32;
    // bytes between consecutive positions, and the lane's own offset
    static constexpr int PITCH_B = RAW ? C::PIXB : kPitchL * 8;
    static AVS_FN int lane_off_b(int lane) {
        return RAW ? (lane >> 1) * C::LINE_B + (lane & 1) * (C::PIXB / 2) : lane * 8;
    }
    // the lane's channel pair at `p`; integer pixels convert exactly ((float) cast); cv: what the
    // sRGB source needs (table, alpha multiplier, whether each of the lane's two channels is alpha)
    static AVS_FN float2 load(const unsigned char* p, const SrcConv& cv) {
        if (SRCT == kSrcU8Srgb) {
            const unsigned v = *reinterpret_cast<const unsigned short*>(p);
            const unsigned b0 = v & 255u, b1 = v >> 8;
            // packScanline with UseSRGBGamma (avir.h:2843-2931): table for colour, (float) b * gm for alpha
            return make_float2(cv.alpha0 ? __fmul_rn((float)b0, cv.gm) : cv.lut[b0],
                               cv.alpha1 ? __fmul_rn((float)b1, cv.gm) : cv.lut[b1]);
        }
        if (SRCT == AVIRB200_U8) {
            const unsigned v = *reinterpret_cast<const unsigned short*>(p);
#if defined(__CUDACC__)
            // byte b -> bits of 2^23 + b (mantissa insert), minus 2^23: exact, no I2F
            return make_float2(__fsub_rn(__uint_as_float(__byte_perm(v, 0x4B000000u, 0x7540)), 8388608.0f),
                               __fsub_rn(__uint_as_float(__byte_perm(v, 0x4B000000u, 0x7541)), 8388608.0f));
#else
            return make_float2((float)(v & 255u), (float)(v >> 8));
#endif
        }
        if (SRCT == AVIRB200_U16) {
            const unsigned v = *reinterpret_cast<const unsigned*>(p);
#if defined(__CUDACC__)
            return make_float2(__fsub_rn(__uint_as_float(__byte_perm(v, 0x4B000000u, 0x7410)), 8388608.0f),
                               __fsub_rn(__uint_as_float(__byte_perm(v, 0x4B000000u, 0x7432)), 8388608.0f));
#else
            return make_float2((float)(v & 65535u), (float)(v >> 16));
#endif
        }
        return *reinterpret_cast<const float2*>(p);
    }
};

// ---- source loader: one group of SRC_N positions, 16 positions x 16 lines per sweep --------------

template <class C, bool IS_V>
AVS_FN void loader_init(const StreamParams& p, WarpRun<C, IS_V>& w) {
    constexpr int PIXB = IS_V ? 16 : C::PIXB;
    const unsigned char* src = static_cast<const unsigned char*>(p.src);
    const size_t rowb = (size_t)p.src_pitch * (PIXB / 4); // bytes between rows (pitch is in elements)
    const int lane = w.lane;
    if constexpr (C::MBAR) return; // the checked rounds compute every address afresh, the tensor copies take coordinates
#pragma unroll
    for (int k = 0; k < C::NK; ++k) {
        if (IS_V) {
            const int piece = lane & 15, rsub = lane >> 4;
            w.gp[k] = src + (ptrdiff_t)(w.o0 - C::POSW + rsub + 2 * k - p.src_row_base) * (ptrdiff_t)rowb +
                      (size_t)(w.line0 + imin_(piece, w.nlines - 1)) * 16;
        } else {
            constexpr int LSTEP = 32 / C::POSW; // lines one pass of the lanes covers
            const int pos = lane & (C::POSW - 1), lsub = lane / C::POSW;
            w.gp[k] = src + (size_t)(w.line0 + imin_(lsub + LSTEP * k, w.nlines - 1)) * rowb +
                      (ptrdiff_t)(w.o0 - C::POSW + pos) * PIXB;
        }
    }
}

// Issues source group g (must be called for g = 0, 1, 2, ... in order: the pointers advance).
// STEADY: the caller guarantees that every sweep is interior (no clamping); `issue` is then a
// uniform predicate of the copies (false in the last rounds of a run, whose groups lie behind it).
template <class C, bool IS_V, bool STEADY>
AVS_FN void load_group(const StreamParams& p, WarpRun<C, IS_V>& w, int g, int gslot, bool issue) {
    constexpr int PITCH_B = RingOf<C, IS_V, 0>::PITCH_B;
    constexpr int PIXB = IS_V ? 16 : C::PIXB;
    const int lane = w.lane;
    const unsigned char* src = static_cast<const unsigned char*>(p.src);
    const size_t rowb = (size_t)p.src_pitch * (PIXB / 4);
    constexpr int POSW = C::POSW, NK = C::NK;
#pragma unroll
    for (int q = 0; q < C::SRC_N / POSW; ++q) {
        const int pos0 = w.o0 + g * C::SRC_N + q * POSW; // first source position of the sweep
        unsigned char* ring = reinterpret_cast<unsigned char*>(w.ring0) + (size_t)(gslot + q * POSW) * PITCH_B;
        const bool interior = STEADY || ((pos0 >= p.src_lo) && (pos0 + POSW <= p.src_hi) &&
                                         (!IS_V || p.xr_flags == nullptr || (pos0 >= p.xr_own_lo && pos0 + POSW <= p.xr_own_hi)));
        if (IS_V) {
            // a position is an intermediate row; the warp's 16 pixel columns are 256 contiguous bytes
            const int piece = lane & 15, rsub = lane >> 4;
            unsigned char* d = ring + rsub * PITCH_B + piece * 16;
            if constexpr (!C::MBAR) {
#pragma unroll
                for (int k = 0; k < NK; ++k) w.gp[k] += POSW * rowb;
            }
            if (!C::MBAR && issue && interior) {
#pragma unroll
                for (int k = 0; k < NK; ++k) cp_async16(d + 2 * k * PITCH_B, w.gp[k]);
            } else if (issue) {
                const size_t coff = (size_t)(w.line0 + imin_(piece, w.nlines - 1)) * 16;
                const unsigned char* col = src + coff;
#pragma unroll
                for (int k = 0; k < NK; ++k) {
                    const int yg = imin_(imax_(pos0 + rsub + 2 * k, p.src_lo), p.src_hi - 1);
                    const unsigned char* g = col + (ptrdiff_t)(yg - p.src_row_base) * (ptrdiff_t)rowb;
                    if (p.xr_flags != nullptr) { // fused halo exchange: the neighbours' rows, in place in the mailbox
                        if (yg < p.xr_own_lo)
                            g = reinterpret_cast<const unsigned char*>(p.xr_up_src) + coff + (size_t)(yg - p.src_lo) * rowb;
                        else if (yg >= p.xr_own_hi)
                            g = reinterpret_cast<const unsigned char*>(p.xr_dn_src) + coff + (size_t)(yg - p.xr_own_hi) * rowb;
                    }
                    cp_async16(d + 2 * k * PITCH_B, g);
                }
            }
        } else {
            // a position is a pixel of a row: POSW consecutive pixels of one row per group of lanes
            constexpr int LSTEP = 32 / POSW;
            const int pos = lane & (POSW - 1), lsub = lane / POSW;
            unsigned char* d = ring + pos * PIXB + lsub * C::LINE_B; // line lsub + LSTEP k: + LSTEP k * LINE_B
            if constexpr (!C::MBAR) {
#pragma unroll
                for (int k = 0; k < NK; ++k) w.gp[k] += POSW * PIXB;
            }
            if (!C::MBAR && issue && interior) {
#pragma unroll
                for (int k = 0; k < NK; ++k) cp_async_px<PIXB>(d + LSTEP * k * C::LINE_B, w.gp[k]);
            } else if (issue) {
                const int x = imin_(imax_(pos0 + pos, p.src_lo), p.src_hi - 1);
#pragma unroll
                for (int k = 0; k < NK; ++k) {
                    const int line = imin_(lsub + LSTEP * k, w.nlines - 1);
                    cp_async_px<PIXB>(d + LSTEP * k * C::LINE_B, src + (size_t)(w.line0 + line) * rowb + (size_t)x * PIXB);
                }
            }
        }
    }
}

// ---- per-output path for batches at the ends of a line ------------------------------------------------
// Reads the input ring by absolute position, each tap clamped to [lo, hi].

template <class C, bool IS_V, int I, class S>
AVS_FN float2 slow_one(const StreamStep& sp, const SrcConv& cv, const unsigned char* ring, int origin, int j, int lo, int hi) {
    using R = RingOf<C, IS_V, I>;
    constexpr int RSP = R::RSP;
    float2 x[S::NTW];
    const int p0 = in_first<S>(sp, j);
#pragma unroll
    for (int t = 0; t < S::NTW; ++t) {
        const int pos = imin_(imax_(p0 + t, lo), hi);
        x[t] = R::load(ring + (size_t)((unsigned)(pos - origin) % (unsigned)RSP) * R::PITCH_B, cv);
    }
    if (S::KIND == K_FIR) return fir_one<S>(x, 0, sp.taps);
    if (S::KIND == K_RESIZE) return resize_one<S>(x, 0, sp.taps, sp.zero_start);
    const int pv = sp.sp_first + j - (S::NT / 2 - 1);
    return (pv & 1) ? resize2_one<S>(x, 0, 1, sp.taps, sp.zero_start)
                    : resize2_one<S>(x, 0, 0, sp.taps, sp.zero_start);
}

// ---- final outputs -------------------------------------------------------------------------------------

// Column pass: lane = (pixel column, channel pair); a batch is M destination rows.
template <int EPI>
AVS_FN void store_v(const StreamParams& p, unsigned char* g, float2 v, int c0, bool gamma_done = false) {
    if (EPI == 1) { // float destination, no output gamma
        *reinterpret_cast<float2*>(g) = v;
        return;
    }
    if (EPI == 2) {
        // integer destination, no output gamma, no bit-depth truncation (stream_epilogue_code()):
        // one rounding conversion per sample, clamp and narrow in integers -- the values of round,
        // clamp, (Tout) in floats -- and no branch: rounding flavour and element size are selects
        // and predicated stores (branches at every store site cost this pass 40 %, profiles/r02a_u8k_ncu_summary.txt)
        const int pk = (int)p.pk_out;
        const int a = imin_(imax_(round_out_int(v.x, p.round_mode), 0), pk);
        const int b = imin_(imax_(round_out_int(v.y, p.round_mode), 0), pk);
        const bool narrow = (p.dst_type == AVIRB200_U8);
        if (narrow) *reinterpret_cast<unsigned short*>(g) = (unsigned short)(a | (b << 8));
        if (!narrow) *reinterpret_cast<unsigned*>(g) = (unsigned)a | ((unsigned)b << 16);
        return;
    }
    v.x = epilogue_value(p, v.x, c0, gamma_done);
    v.y = epilogue_value(p, v.y, c0 + 1, gamma_done);
    if (p.dst_type == AVIRB200_F32) *reinterpret_cast<float2*>(g) = v;
    else if (p.dst_type == AVIRB200_U8)
        *reinterpret_cast<uchar2*>(g) = make_uchar2((unsigned char)v.x, (unsigned char)v.y);
    else
        *reinterpret_cast<ushort2*>(g) = make_ushort2((unsigned short)v.x, (unsigned short)v.y);
}

template <class C, int EPI, int M, bool STEADY>
AVS_FN void sink_v(const StreamParams& p, const WarpRun<C, true>& w, int j0, const float2* o) {
    const int q = w.lane >> 1, c0 = (w.lane & 1) * 2;
    if (q >= w.nlines) return;
    const size_t esz = (p.dst_type == AVIRB200_F32) ? 4 : (p.dst_type == AVIRB200_U16 ? 2 : 1);
    const size_t rowb = (size_t)p.dst_pitch * esz;
    unsigned char* g = static_cast<unsigned char*>(p.dst) + ((size_t)(w.line0 + q) * 4 + c0) * esz +
                       (ptrdiff_t)(j0 - p.dst_row_base) * (ptrdiff_t)rowb;
    if constexpr (EPI == 0) {
        // the run-time output stage: gamma for the whole batch first (when the plan has one)
        float2 t[M];
#pragma unroll
        for (int m = 0; m < M; ++m) t[m] = o[m];
        const bool gamma_done = p.gamma_out && epilogue_gamma_batch<M>(p, t, c0);
#pragma unroll
        for (int m = 0; m < M; ++m) {
            if (STEADY || (j0 + m >= p.out0 && j0 + m < p.out1)) store_v<EPI>(p, g, t[m], c0, gamma_done);
            g += rowb;
        }
        return;
    }
    if (STEADY || (j0 >= p.out0 && j0 + M <= p.out1)) {
#pragma unroll
        for (int m = 0; m < M; ++m) {
            store_v<EPI>(p, g, o[m], c0);
            g += rowb;
        }
    } else {
#pragma unroll
        for (int m = 0; m < M; ++m) {
            if (j0 + m >= p.out0 && j0 + m < p.out1) store_v<EPI>(p, g, o[m], c0);
            g += rowb;
        }
    }
}

// Row pass: lanes hold (line, channel pair) of M consecutive pixels; transposed through the
// staging rows so that every store instruction writes runs of whole pixels of a row.  The
// read-back of batch b is issued before batch b+1 is computed and its global stores after,
// so that neither the shared-memory latency nor the stores' operand reads are waited for.
constexpr int kNoPend = -0x7fffffff;

template <class C, int M>
AVS_FN void sink_h_readback(WarpRun<C, false>& w) {
    // unconditional (no branch around the loads: a join would wait for them); without a
    // pending batch the values are never stored
    const int pos = w.lane & (M - 1), lsub = w.lane / M;
#pragma unroll
    for (int k = 0; k < M / 2; ++k)
        w.pend[k] = *reinterpret_cast<const float4*>(w.stage + (lsub + (32 / M) * k) * C::STAGE_LINE + pos * 2);
}

// XS: the row pass of a sharded band with the fused halo exchange (its own instantiation, kEpiXs: the
// plain kernel's loop carries none of it).
template <class C, int M, bool XS = false>
AVS_FN void sink_h_store(const StreamParams& p, WarpRun<C, false>& w) {
    const int pos = w.lane & (M - 1), lsub = w.lane / M;
    const int j = w.pend_j0 + pos;
    float* dst = static_cast<float*>(p.dst);
    const bool jok = (w.pend_j0 != kNoPend) && (j >= p.out0) && (j < p.out1);
    float4* g = reinterpret_cast<float4*>(dst + (size_t)(w.line0 + lsub) * (size_t)p.dst_pitch) + j;
    const size_t gstep = (size_t)(32 / M) * (size_t)(p.dst_pitch / 4);
#pragma unroll
    for (int k = 0; k < M / 2; ++k) {
        if (jok && lsub + (32 / M) * k < w.nlines) *g = w.pend[k];
        g += gstep;
    }
    if constexpr (XS) {
        // fused halo exchange: the lines [xs_l0, xs_l1) of this strip (empty outside the first / last strips of
        // a sharded band) also go straight into a neighbour's mailbox -- peer memory over NVLink, xs_delta
        // bytes from the line's own address.  Predicated stores, no branch: the loop stays straight-line.
        unsigned char* ga = reinterpret_cast<unsigned char*>(reinterpret_cast<float4*>(dst + (size_t)(w.line0 + lsub) * (size_t)p.dst_pitch) + j) + w.xs_delta;
#pragma unroll
        for (int k = 0; k < M / 2; ++k) {
            const int l = lsub + (32 / M) * k;
            if (jok && l >= w.xs_l0 && l < w.xs_l1) *reinterpret_cast<float4*>(ga) = w.pend[k];
            ga += gstep * sizeof(float4);
        }
    }
    w.pend_j0 = kNoPend;
}

template <class C, int M>
AVS_FN void sink_h_stage(WarpRun<C, false>& w, int j0, const float2* o) {
    AVS_SYNCWARP(); // every lane has read the previous batch back
#pragma unroll
    for (int m = 0; m < M; ++m) w.stage[(w.lane >> 1) * C::STAGE_LINE + m * 2 + (w.lane & 1)] = o[m];
    AVS_SYNCWARP();
    w.pend_j0 = j0;
}

// ---- one batch of one step ------------------------------------------------------------------------------

// Outputs of one in-domain batch whose whole window lies inside its input line.
template <class C, bool IS_V, int I, class S>
AVS_FN void window_bases(const unsigned char* ring, int rd, const unsigned char** base) {
    constexpr int RSP = RingOf<C, IS_V, I>::RSP;
    constexpr int PITCH_B = RingOf<C, IS_V, I>::PITCH_B;
    // the window never wraps inside a piece of CH positions: pieces are ring-aligned
#pragma unroll
    for (int k = 0; k < (S::W + S::CH - 1) / S::CH; ++k) {
        int s = rd + k * S::CH;
        if (s >= RSP) s -= RSP;
        base[k] = ring + (size_t)s * PITCH_B;
    }
}

template <class C, bool IS_V, int I, class S>
AVS_FN void fast_batch(const StreamParams& p, WarpRun<C, IS_V>& w, const unsigned char* ring, int rd, int kbcur,
                       int j0, float2* o) {
    using R = RingOf<C, IS_V, I>;
    constexpr int PITCH_B = R::PITCH_B;
    constexpr int M = S::M;
    const StreamStep& sp = p.s[I];
    const unsigned char* base[(S::W + S::CH - 1) / S::CH + 1];
    window_bases<C, IS_V, I, S>(ring, rd, base);
    if constexpr (S::KIND == K_RESIZE2) {
        float2 x[S::W];
#pragma unroll
        for (int i = 0; i < S::W; ++i) x[i] = R::load(base[i / S::CH] + (i % S::CH) * PITCH_B, w.cv);
        const int pv = sp.sp_first + j0 - (S::NT / 2 - 1);
        if (pv & 1) {
#pragma unroll
            for (int m = 0; m < M; ++m) o[m] = resize2_one<S>(x, m >> 1, (m & 1) ? 0 : 1, sp.taps, sp.zero_start);
        } else {
#pragma unroll
            for (int m = 0; m < M; ++m) o[m] = resize2_one<S>(x, (m + 1) >> 1, m & 1, sp.taps, sp.zero_start);
        }
    } else if constexpr (S::KIND == K_RESIZE && S::SUM == AVIRB200_SUM_DIL8 && (S::NT > 32)) {
        // long filter: the window (NT + (M-1)*ADV positions) does not fit the register file next to
        // the M x 8 lane sums; walk the taps in their groups of 8 (the order resize_one() adds them
        // in anyway) and read each group's inputs when it is their turn
        const StreamTap* t = sp.taps;
        const StreamTap& one = t[kTapOne];
        float2 ln[M][8];
#pragma unroll
        for (int g = 0; g < S::NT / 8; ++g) {
            constexpr int GW = (M - 1) * S::ADV + 8;
            float2 xg[GW];
#pragma unroll
            for (int i = 0; i < GW; ++i) {
                const int pos = g * 8 + i;
                xg[i] = R::load(base[pos / S::CH] + (pos % S::CH) * PITCH_B, w.cv);
            }
#pragma unroll
            for (int m = 0; m < M; ++m) {
#pragma unroll
                for (int q = 0; q < 8; ++q) {
                    const float2 v = f2mul(t[g * 8 + q], xg[m * S::ADV + q]);
                    ln[m][q] = (g == 0) ? v : f2add(ln[m][q], v, one);
                }
            }
        }
#pragma unroll
        for (int m = 0; m < M; ++m) {
            o[m] = f2hadd8(ln[m], one);
            if (sp.zero_start) o[m] = f2add(o[m], make_float2(0.0f, 0.0f), one);
        }
    } else {
        // whole window of the batch in registers
        float2 x[S::W];
#pragma unroll
        for (int i = 0; i < S::W; ++i) x[i] = R::load(base[i / S::CH] + (i % S::CH) * PITCH_B, w.cv);
#pragma unroll
        for (int m = 0; m < M; ++m) {
            if (S::KIND == K_FIR) o[m] = fir_one<S>(x, m * S::ADV, sp.taps);
            else o[m] = resize_one<S>(x, m * S::ADV, sp.taps, sp.zero_start);
        }
    }
}

// STEADY: the batch is known to be in-domain with its window inside the input line and (last
// step) its outputs inside [out0, out1): straight-line code, no checks.
template <class C, bool IS_V, int EPI, int I, class S, bool STEADY>
AVS_FN void run_batch(const StreamParams& p, WarpRun<C, IS_V>& w) {
    constexpr bool LAST = (I == C::NS - 1);
    constexpr int RSP = RingOf<C, IS_V, I>::RSP;
    constexpr int M = S::M;
    const StreamStep& sp = p.s[I];
    const int kbcur = w.kb[I];
    const int j0 = w.a[I] + M * kbcur;
    const unsigned char* ring = reinterpret_cast<const unsigned char*>((I == 0) ? w.ring0 : (I == 1 ? w.ring1 : w.ring2)) +
                                RingOf<C, IS_V, I>::lane_off_b(w.lane);
    const int origin = (I == 0) ? w.o0 : w.a[I - 1];
    const int rd = w.rd[I];
    const int wr = w.wr[I];
    // advance the ring cursors first (uniform bookkeeping, also for skipped batches)
    w.kb[I] += 1;
    w.rd[I] = (rd + S::CH == RSP) ? 0 : rd + S::CH;

    if constexpr (LAST && !IS_V) sink_h_readback<C, M>(w);
    float2 o[M];
    bool have = true;
    if constexpr (STEADY) {
        fast_batch<C, IS_V, I, S>(p, w, ring, rd, kbcur, j0, o);
    } else {
        const int pin = in_first<S>(sp, j0);
        const bool in_dom = (j0 >= 0) && (j0 + M <= sp.out_len);
        const bool win_ok = (I == 0) || (pin >= 0 && pin + S::W <= sp.in_len);
        if (j0 + M <= 0 || j0 >= sp.out_len) {
            have = false; // nothing of this batch exists
        } else if (in_dom && win_ok) {
            fast_batch<C, IS_V, I, S>(p, w, ring, rd, kbcur, j0, o);
        } else {
            const int lo = (I == 0) ? -0x40000000 : 0;
            const int hi = (I == 0) ? 0x40000000 : sp.in_len - 1;
#pragma unroll 1
            for (int m = 0; m < M; ++m) {
                const int j = j0 + m;
                float2 v = make_float2(0.0f, 0.0f);
                if (j >= 0 && j < sp.out_len) v = slow_one<C, IS_V, I, S>(sp, w.cv, ring, origin, j, lo, hi);
                // (a register array indexed by the loop counter: keep the loop rolled, select by value)
#pragma unroll
                for (int mm = 0; mm < M; ++mm)
                    if (mm == m) o[mm] = v;
            }
        }
    }

    if constexpr (!LAST) {
        constexpr int RSPO = RingOf<C, IS_V, I + 1>::RSP;
        constexpr int PITCHO = kPitchL; // intermediate rings: float2 [position][lane]
        w.wr[I] = (wr + M == RSPO) ? 0 : wr + M;
        if (STEADY || have) {
            float2* out = ((I == 0) ? w.ring1 : w.ring2) + w.lane + (size_t)wr * PITCHO;
#pragma unroll
            for (int m = 0; m < M; ++m) out[m * PITCHO] = o[m];
        }
    } else if constexpr (IS_V) {
        if (STEADY || have) sink_v<C, EPI, M, STEADY>(p, w, j0, o);
    } else {
        sink_h_store<C, M, EPI == kEpiXs>(p, w);
        if (STEADY || have) sink_h_stage<C, M>(w, j0, o);
    }
}

// Rounds [lo, hi] of a run in which step I's batches all satisfy the STEADY conditions.
AVS_FN int fdiv_(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }
AVS_FN int cdiv_(int a, int b) { return -fdiv_(-a, b); }

template <class C, bool IS_V, int I, class S>
AVS_FN void steady_bounds(const StreamParams& p, const WarpRun<C, IS_V>& w, int delay, int reps, int& lo, int& hi) {
    constexpr bool LAST = (I == C::NS - 1);
    const StreamStep& sp = p.s[I];
    int kb_lo = imax_(0, cdiv_(-w.a[I], S::M));
    int kb_hi = fdiv_(sp.out_len - S::M - w.a[I], S::M);
    if (I > 0) {
        const int pin0 = in_first<S>(sp, w.a[I]); // window of batch kb starts at pin0 + CH * kb
        kb_lo = imax_(kb_lo, cdiv_(-pin0, S::CH));
        kb_hi = imin_(kb_hi, fdiv_(sp.in_len - S::W - pin0, S::CH));
    }
    if (LAST) {
        kb_lo = imax_(kb_lo, cdiv_(p.out0 - w.a[I], S::M));
        kb_hi = imin_(kb_hi, fdiv_(p.out1 - S::M - w.a[I], S::M));
    }
    lo = imax_(lo, delay + cdiv_(kb_lo, reps));
    hi = imin_(hi, delay + fdiv_(kb_hi - reps + 1, reps));
}

// ---- register-window rounds (C::REGWIN) -----------------------------------------------------------------
// The ring rounds above read every batch's whole window from shared memory (38 reads per 8
// outputs of the 24-tap resize, the later steps through their own rings) and wait for it
// before the arithmetic starts; with two warps per scheduler those waits show (stall `wait` +
// `long scoreboard`, FP32 pipe 74 % busy, profiles/r01_final_ncu_summary.txt).  In the interior
// of a run the windows slide through REGISTERS instead: every round reads only the SRC_N source
// positions it has not seen yet -- they are first needed by the round's last outputs, so the
// shared-memory latency hides behind the arithmetic of the first ones -- and a later step's window
// is the previous step's outputs, which never leave the register file.  Shared memory then
// carries the source ring only (one read per input) plus the row pass's output staging.
//
// win0[q]: source position (first position of the round's step-0 window) + q; win1 / win2: the
// same for steps 1 / 2, whose producers append this round's outputs at d * A (the consumer lags
// d rounds).  After its arithmetic a window shifts down by the positions the step consumed: in
// the unrolled loop that is register renaming.  Entering, the windows are filled from the
// rings the checked rounds wrote; leaving, the later steps' windows are written back so that
// the checked rounds can go on.
template <class C>
struct RegWinGeom {
    using S0 = typename C::T0;
    using S1 = typename C::T1;
    using S2 = typename C::T2;
    static constexpr int A0 = C::SRC_N;                           // positions a round consumes
    static constexpr int WR0 = S0::W + (C::reps0 - 1) * S0::CH;   // positions a round reads
    static constexpr int Q0 = WR0 - A0;                           // first position a round has not seen before
    static constexpr int A1 = S1::CH * C::reps1;
    static constexpr int WR1 = S1::W + (C::reps1 - 1) * S1::CH;
    static constexpr int K1 = C::d0 * A1;                         // positions kept from earlier rounds
    static constexpr int A2 = (C::NS == 3) ? S2::CH * C::reps2 : 1;
    static constexpr int WR2 = (C::NS == 3) ? S2::W + (C::reps2 - 1) * S2::CH : 1;
    static constexpr int K2 = (C::NS == 3) ? C::d1 * A2 : 0;
    static_assert(S0::M * C::reps0 == A1, "step 0 outputs per round");
    static_assert(C::NS == 2 || S1::M * C::reps1 == A2, "step 1 outputs per round");
    static_assert(WR1 <= K1 + A1 && WR2 <= K2 + A2, "window inside the kept positions");
    static_assert(Q0 < C::rsp0 && Q0 >= 0, "source window");
};

template <class C>
struct RegWin {
    using G = RegWinGeom<C>;
    float2 w0[G::WR0];
    float2 w1[G::K1 + G::A1];
    float2 w2[G::K2 + G::A2];
};

template <class S, class X>
AVS_FN float2 step_one(const X& x, const int off, const StreamStep& sp) {
    if (S::KIND == K_FIR) return fir_one<S>(x, off, sp.taps);
    return resize_one<S>(x, off, sp.taps, sp.zero_start);
}

template <class C, bool IS_V>
AVS_FN void regwin_enter(const WarpRun<C, IS_V>& w, RegWin<C>& R) {
    using G = RegWinGeom<C>;
    using R0 = RingOf<C, IS_V, 0>;
    const unsigned char* ring0 = reinterpret_cast<const unsigned char*>(w.ring0) + R0::lane_off_b(w.lane);
#pragma unroll
    for (int q = 0; q < G::Q0; ++q) {
        int s = w.rd[0] + q;
        if (s >= C::rsp0) s -= C::rsp0;
        R.w0[q] = R0::load(ring0 + (size_t)s * R0::PITCH_B, w.cv);
    }
#pragma unroll
    for (int q = 0; q < G::K1; ++q) {
        int s = w.rd[1] + q;
        if (s >= C::rsp1) s -= C::rsp1;
        R.w1[q] = w.ring1[(size_t)s * kPitchL + w.lane];
    }
    if constexpr (C::NS == 3) {
#pragma unroll
        for (int q = 0; q < G::K2; ++q) {
            int s = w.rd[2] + q;
            if (s >= C::rsp2) s -= C::rsp2;
            R.w2[q] = w.ring2[(size_t)s * kPitchL + w.lane];
        }
    }
}

// n rounds were run in registers: advance the ring cursors as the ring rounds would have and
// write the kept part of the later steps' windows where the next checked round reads it.
template <class C, bool IS_V>
AVS_FN void regwin_leave(WarpRun<C, IS_V>& w, const RegWin<C>& R, int n) {
    using G = RegWinGeom<C>;
    w.rd[0] = (int)(((unsigned)w.rd[0] + (unsigned)n * G::A0) % (unsigned)C::rsp0);
    w.kb[0] += n * C::reps0;
    w.wr[0] = (int)(((unsigned)w.wr[0] + (unsigned)n * G::A1) % (unsigned)C::rsp1);
    w.rd[1] = (int)(((unsigned)w.rd[1] + (unsigned)n * G::A1) % (unsigned)C::rsp1);
    w.kb[1] += n * C::reps1;
#pragma unroll
    for (int q = 0; q < G::K1; ++q) {
        int s = w.rd[1] + q;
        if (s >= C::rsp1) s -= C::rsp1;
        w.ring1[(size_t)s * kPitchL + w.lane] = R.w1[q];
    }
    if constexpr (C::NS == 3) {
        w.wr[1] = (int)(((unsigned)w.wr[1] + (unsigned)n * G::A2) % (unsigned)C::rsp2);
        w.rd[2] = (int)(((unsigned)w.rd[2] + (unsigned)n * G::A2) % (unsigned)C::rsp2);
        w.kb[2] += n * C::reps2;
#pragma unroll
        for (int q = 0; q < G::K2; ++q) {
            int s = w.rd[2] + q;
            if (s >= C::rsp2) s -= C::rsp2;
            w.ring2[(size_t)s * kPitchL + w.lane] = R.w2[q];
        }
    }
}

// Stages source group g of the column pass (interior: no clamping) with ONE tensor copy issued
// by one lane: the box SRC_N intermediate rows x 256 bytes (the strip's 16 pixel columns) lands
// as the ring's [position][lane] rows.  Columns past the image's right edge (ragged strip) are
// outside the tensor: the TMA unit fills them with zeros, their lanes never store.
template <class C, bool IS_V>
AVS_FN void bulk_group(const StreamParams& p, WarpRun<C, IS_V>& w, int row, int gslot, unsigned bar) {
    static_assert(IS_V, "tensor staging: column pass");
    unsigned char* d = reinterpret_cast<unsigned char*>(w.ring0) + (size_t)gslot * (kPitchL * 8);
#if defined(__CUDACC__)
    if (w.lane == 0) {
        mbar_arrive_expect_tx(bar, C::SRC_N * kPitchL * 8);
        tma_tile_2d(d, &p.tmap, w.line0 * 4, row, bar);
    } else {
        mbar_arrive(bar);
    }
#else
    if (w.lane == 0) {
        const unsigned char* src = static_cast<const unsigned char*>(p.src);
        const size_t rowb = (size_t)p.src_pitch * 4;
        for (int k = 0; k < C::SRC_N; ++k)
            emul_copy(d + k * (kPitchL * 8), src + (size_t)(row + k) * rowb + (size_t)w.line0 * 16, w.nlines * 16);
    }
    (void)bar;
#endif
}

// One round in registers.  s1 / s2: ring slots (positions) of the two source groups the round's
// new positions lie in; jout: first final output of the round.
template <class C, bool IS_V, int EPI>
AVS_FN void regwin_round(const StreamParams& p, WarpRun<C, IS_V>& w, RegWin<C>& R, int s1, int s2, int jout) {
    using G = RegWinGeom<C>;
    using S0 = typename C::T0;
    using S1 = typename C::T1;
    using S2 = typename C::T2;
    using R0 = RingOf<C, IS_V, 0>;
    constexpr int OQ = G::Q0 % G::A0; // offset of the first new position inside its group
    const unsigned char* ring0 = reinterpret_cast<const unsigned char*>(w.ring0) + R0::lane_off_b(w.lane);
    const unsigned char* b1 = ring0 + (size_t)s1 * R0::PITCH_B;
    const unsigned char* b2 = ring0 + (size_t)s2 * R0::PITCH_B;
#pragma unroll
    for (int i = 0; i < G::A0; ++i) {
        R.w0[G::Q0 + i] = (i < G::A0 - OQ) ? R0::load(b1 + (OQ + i) * R0::PITCH_B, w.cv)
                                           : R0::load(b2 + (i - (G::A0 - OQ)) * R0::PITCH_B, w.cv);
    }
    float2 o[C::B];
    // step 0
#pragma unroll
    for (int q = 0; q < C::reps0; ++q) {
#pragma unroll
        for (int m = 0; m < S0::M; ++m)
            R.w1[G::K1 + q * S0::M + m] = step_one<S0>(R.w0, q * S0::CH + m * S0::ADV, p.s[0]);
    }
#pragma unroll
    for (int k = 0; k < G::Q0; ++k) R.w0[k] = R.w0[k + G::A0];
    // step 1
#pragma unroll
    for (int q = 0; q < C::reps1; ++q) {
#pragma unroll
        for (int m = 0; m < S1::M; ++m) {
            const float2 v = step_one<S1>(R.w1, q * S1::CH + m * S1::ADV, p.s[1]);
            if constexpr (C::NS == 3) R.w2[G::K2 + q * S1::M + m] = v;
            else o[q * S1::M + m] = v;
        }
    }
#pragma unroll
    for (int k = 0; k < G::K1; ++k) R.w1[k] = R.w1[k + G::A1];
    if constexpr (C::NS == 3) {
#pragma unroll
        for (int q = 0; q < C::reps2; ++q) {
#pragma unroll
            for (int m = 0; m < S2::M; ++m) o[q * S2::M + m] = step_one<S2>(R.w2, q * S2::CH + m * S2::ADV, p.s[2]);
        }
#pragma unroll
        for (int k = 0; k < G::K2; ++k) R.w2[k] = R.w2[k + G::A2];
    }
    // final outputs (every batch inside [out0, out1): steady_bounds)
    constexpr int ML = C::MLAST;
#pragma unroll
    for (int q = 0; q < C::B / ML; ++q) {
        if constexpr (IS_V) {
            sink_v<C, EPI, ML, true>(p, w, jout + q * ML, o + q * ML);
        } else {
            if (q > 0) sink_h_readback<C, ML>(w);
            sink_h_store<C, ML, EPI == kEpiXs>(p, w);
            sink_h_stage<C, ML>(w, jout + q * ML, o + q * ML);
        }
    }
}

// Rounds [r, r + n) of a run in registers (n a multiple of C::RW_UNROLL, every round "steady").
// gslot / gi: ring slot (positions / group index) the loader fills next; wi: group index the
// next round waits for (C::MBAR).
template <class C, bool IS_V, int EPI>
AVS_FN void run_regwin(const StreamParams& p, WarpRun<C, IS_V>& w, int r, int n, int groups, int& gslot, int& gi, int& wi) {
    using G = RegWinGeom<C>;
    constexpr int PRO = C::H + C::LOOKAHEAD;
    RegWin<C> R;
    regwin_enter<C, IS_V>(w, R);
    int s1 = w.rd[0] + (G::Q0 / G::A0) * G::A0;
    if (s1 >= C::rsp0) s1 -= C::rsp0;
    int s2 = (s1 + G::A0 == C::rsp0) ? 0 : s1 + G::A0;
    int jout = w.a[C::NS - 1] + C::MLAST * w.kb[C::NS - 1];
    int grow = w.o0 + (r + PRO) * C::SRC_N - p.src_row_base; // C::MBAR: first buffer row of the group staged next
    for (int it = n / C::RW_UNROLL; it > 0; --it) {
#pragma unroll
        for (int u = 0; u < C::RW_UNROLL; ++u) {
            if constexpr (C::MBAR) {
                mbar_wait(w.mbar0 + wi * 8, (w.mpar >> wi) & 1u);
                w.mpar ^= 1u << wi;
                wi = (wi + 1 == C::NG) ? 0 : wi + 1;
            } else {
                cp_async_wait<C::LOOKAHEAD - 1>();
            }
            AVS_SYNCWARP(); // all lanes' copies have landed; the previous round is done with its slots
            if constexpr (!IS_V) sink_h_readback<C, C::MLAST>(w);
            const bool issue = (r + PRO < groups); // (the last rounds of a run issue nothing)
            if constexpr (C::MBAR) {
                if (issue) bulk_group<C, IS_V>(p, w, grow, gslot, w.mbar0 + gi * 8);
                grow += C::SRC_N;
                gi = (gi + 1 == C::NG) ? 0 : gi + 1;
            } else {
                load_group<C, IS_V, true>(p, w, r + PRO, gslot, issue);
                cp_async_commit();
            }
            gslot = (gslot + C::SRC_N == C::rsp0) ? 0 : gslot + C::SRC_N;
            regwin_round<C, IS_V, EPI>(p, w, R, s1, s2, jout);
            s1 = s2;
            s2 = (s2 + G::A0 == C::rsp0) ? 0 : s2 + G::A0;
            jout += C::B;
            ++r;
        }
    }
    regwin_leave<C, IS_V>(w, R, n);
}

// ---- one run: `rounds` rounds of B final outputs of one 16-line strip -----------------------------

template <class C, bool IS_V, int EPI>
AVS_FN void run_warp(const StreamParams& p, WarpRun<C, IS_V>& w, int strip, int rho0, int rounds) {
    using S0 = typename C::T0;
    using S1 = typename C::T1;
    using S2 = typename C::T2;
    w.line0 = strip * kLines;
    w.nlines = imin_(kLines, p.n_lines - w.line0);
    if (p.seg_b > 0) { // two segments, each with its own strips (stream_types.h)
        const int sa = (p.seg_a + kLines - 1) / kLines;
        if (strip < sa) {
            w.nlines = imin_(kLines, p.seg_a - w.line0);
        } else {
            w.line0 = p.seg_b_line0 + (strip - sa) * kLines;
            w.nlines = imin_(kLines, p.seg_b_line0 + p.seg_b - w.line0);
        }
    }
    if (C::NS == 3) {
        w.a[2] = C::B * rho0;
        w.a[1] = in_first<S2>(p.s[2], w.a[2]);
    } else {
        w.a[1] = C::B * rho0;
    }
    w.a[0] = in_first<S1>(p.s[1], w.a[1]);
    w.o0 = in_first<S0>(p.s[0], w.a[0]);
#pragma unroll
    for (int i = 0; i < kMaxSteps; ++i) w.rd[i] = w.wr[i] = w.kb[i] = 0;

    const int total = rounds + C::DELAY_LAST;  // wall rounds; step 0 runs all of them
    const int groups = total + C::H;           // source groups step 0 reads
    const bool fused_rx = IS_V && p.xr_flags != nullptr;
    const int int_lo = fused_rx ? p.xr_own_lo : p.src_lo, int_hi = fused_rx ? p.xr_own_hi : p.src_hi;
    if (fused_rx) {
        // fused halo exchange: a run that reads the neighbours' rows waits for them here, once
        const int first = w.o0, last = w.o0 + groups * C::SRC_N;
        if (first < p.xr_own_lo && p.xr_own_lo > p.src_lo) xr_wait(p.xr_flags + 0, p.xr_seq);
        if (last > p.xr_own_hi && p.xr_own_hi < p.src_hi) xr_wait(p.xr_flags + 1, p.xr_seq);
    }
    int gslot = 0;
    int gi = 0, wi = 0; // C::MBAR: group index (ring slot / SRC_N) the loader fills / a round waits for next
    constexpr int PRO = C::H + C::LOOKAHEAD;
    loader_init<C, IS_V>(p, w);
    if constexpr (!IS_V) w.pend_j0 = kNoPend;
    if constexpr (!IS_V) {
        w.xs_l0 = w.xs_l1 = w.xs_dir = 0;
        w.xs_delta = 0;
    }
    if constexpr (!IS_V && EPI == kEpiXs) {
        // (the host launches this kernel only when no strip holds rows of both neighbours)
        const ptrdiff_t rowb = (ptrdiff_t)p.dst_pitch * 4;
        if (p.xs_up_dst != nullptr && w.line0 < p.xs_top) {
            w.xs_l1 = imin_(w.nlines, p.xs_top - w.line0);
            w.xs_delta = reinterpret_cast<const unsigned char*>(p.xs_up_dst) - static_cast<const unsigned char*>(p.dst);
        } else if (p.xs_dn_dst != nullptr && w.line0 + w.nlines > p.xs_bot0 && w.line0 < p.xs_bot0 + p.xs_bot) {
            w.xs_dir = 1;
            w.xs_l0 = imax_(0, p.xs_bot0 - w.line0);
            w.xs_l1 = imin_(w.nlines, p.xs_bot0 + p.xs_bot - w.line0);
            w.xs_delta = reinterpret_cast<const unsigned char*>(p.xs_dn_dst) - static_cast<const unsigned char*>(p.dst) -
                         (ptrdiff_t)p.xs_bot0 * rowb;
        }
    }
    // one checked group: per-lane copies (clamped at the line's ends), completion through the
    // lane's cp.async group or, C::MBAR, the group's mbarrier
#define AVS_ISSUE_CHECKED(G)                                                                          \
    {                                                                                                 \
        const bool issue_ = (G) < groups;                                                             \
        load_group<C, IS_V, false>(p, w, (G), gslot, issue_);                                         \
        if constexpr (C::MBAR) {                                                                      \
            if (issue_) mbar_arrive_cp_async(w.mbar0 + gi * 8);                                       \
            gi = (gi + 1 == C::NG) ? 0 : gi + 1;                                                      \
        } else {                                                                                      \
            cp_async_commit();                                                                        \
        }                                                                                             \
        gslot = (gslot + C::SRC_N == C::rsp0) ? 0 : gslot + C::SRC_N;                                 \
    }
#define AVS_WAIT_GROUP()                                                                              \
    {                                                                                                 \
        mbar_wait(w.mbar0 + wi * 8, (w.mpar >> wi) & 1u);                                             \
        w.mpar ^= 1u << wi;                                                                           \
        wi = (wi + 1 == C::NG) ? 0 : wi + 1;                                                          \
    }
    for (int g = 0; g < PRO; ++g) AVS_ISSUE_CHECKED(g)
    if constexpr (C::MBAR) {
        // round r waits for group r + H; groups 0 .. H-1 have no round of their own
        for (int g = 0; g < C::H; ++g) AVS_WAIT_GROUP()
    }
    // rounds [slo, shi]: every batch of every step and the source group issued are "steady"
    int slo = C::DELAY_LAST, shi = total - 1;
    steady_bounds<C, IS_V, 0, S0>(p, w, C::delay0, C::reps0, slo, shi);
    steady_bounds<C, IS_V, 1, S1>(p, w, C::delay1, C::reps1, slo, shi);
    if constexpr (C::NS == 3) steady_bounds<C, IS_V, 2, S2>(p, w, C::delay2, C::reps2, slo, shi);
    // the group a steady round issues (r + PRO) is interior -- or lies behind the run (not issued)
    slo = imax_(slo, cdiv_(int_lo - w.o0, C::SRC_N) - PRO);
    {
        const int g_int_hi = fdiv_(int_hi - w.o0, C::SRC_N) - 1; // last group without clamping
        if (groups - 1 > g_int_hi) shi = imin_(shi, g_int_hi - PRO);
    }

#define AVS_ROUND(STEADY)                                                                             \
    {                                                                                                 \
        if constexpr (C::MBAR) AVS_WAIT_GROUP()                                                       \
        else cp_async_wait<C::LOOKAHEAD - 1>(); /* groups <= r + H have landed (this lane's copies) */ \
        AVS_SYNCWARP();                    /* ... all lanes'; round r-1 is done with its slots */     \
        if constexpr (STEADY) {                                                                       \
            load_group<C, IS_V, true>(p, w, r + PRO, gslot, r + PRO < groups);                        \
            cp_async_commit();                                                                        \
            gslot = (gslot + C::SRC_N == C::rsp0) ? 0 : gslot + C::SRC_N;                             \
        } else {                                                                                      \
            AVS_ISSUE_CHECKED(r + PRO)                                                                \
        }                                                                                             \
        _Pragma("unroll") for (int q = 0; q < C::reps0; ++q) run_batch<C, IS_V, EPI, 0, S0, STEADY>(p, w); \
        if (STEADY || r >= C::delay1) {                                                               \
            _Pragma("unroll") for (int q = 0; q < C::reps1; ++q) run_batch<C, IS_V, EPI, 1, S1, STEADY>(p, w); \
        }                                                                                             \
        if constexpr (C::NS == 3) {                                                                   \
            if (STEADY || r >= C::delay2) {                                                           \
                _Pragma("unroll") for (int q = 0; q < C::reps2; ++q) run_batch<C, IS_V, EPI, 2, S2, STEADY>(p, w); \
            }                                                                                         \
        }                                                                                             \
    }
    int r = 0;
    while (r < total) {
        if constexpr (C::REGWIN) {
            // the interior of the run in registers; what is left of it (fewer rounds than one
            // trip of the unrolled loop) takes the checked path
            const int n = (shi - r + 1) / C::RW_UNROLL * C::RW_UNROLL;
            if (r == slo && n > 0) {
                run_regwin<C, IS_V, EPI>(p, w, r, n, groups, gslot, gi, wi);
                r += n;
                continue;
            }
            AVS_ROUND(false)
            ++r;
        } else {
            if (C::STEADY_LOOP && r >= slo && r <= shi) {
                // the hot loop: straight-line rounds
                do {
                    AVS_ROUND(true)
                    ++r;
                } while (r <= shi);
            } else {
                AVS_ROUND(false)
                ++r;
            }
        }
    }
#undef AVS_ROUND
#undef AVS_ISSUE_CHECKED
#undef AVS_WAIT_GROUP
    if constexpr (!IS_V) {
        // the last batch is still in the staging rows
        sink_h_readback<C, C::MLAST>(w);
        sink_h_store<C, C::MLAST, EPI == kEpiXs>(p, w);
    }
    if constexpr (!C::MBAR) cp_async_wait<0>(); // (C::MBAR: every issued group has been waited for)
    AVS_SYNCWARP(); // the next run refills the rings
    if constexpr (!IS_V && EPI == kEpiXs) {
        if (w.xs_l1 > w.xs_l0) {
            // fused halo exchange: this run's rows are in the neighbour's mailbox; the warp that
            // completes the call's total of boundary-strip rounds publishes the sequence number
            xs_fence();
            AVS_SYNCWARP();
            if (w.lane == 0) {
                const unsigned long long rps = (unsigned long long)((p.out1 - 1) / C::B - p.out0 / C::B + 1); // rounds per strip
                const unsigned long long done = xs_add(p.xs_count + w.xs_dir, (unsigned long long)rounds) + (unsigned long long)rounds;
                if (done == p.xs_units[w.xs_dir] * rps) {
                    p.xs_count[w.xs_dir] = 0;
                    xs_publish(w.xs_dir ? p.xs_dn_flag : p.xs_up_flag, p.xs_seq);
                }
            }
        }
    }
}

// ---- a warp's share of the pass -------------------------------------------------------------------------
// Units = rounds of B final outputs, strip-major; every warp takes an equal contiguous share.

template <class C, bool IS_V, int EPI>
AVS_FN void stream_warp_main(const StreamParams& p, long long gw, long long nwarps, int lane, float2* sm,
                             const float* lut) {
    WarpRun<C, IS_V> w;
    w.lane = lane;
    w.cv.lut = lut; // (sRGB source only) the linearisation table, in shared memory on the device
    w.cv.gm = p.in_gamma_mult;
    w.cv.alpha0 = (p.alpha_index == (lane & 1) * 2);
    w.cv.alpha1 = (p.alpha_index == (lane & 1) * 2 + 1);
    w.ring0 = sm;
    w.ring1 = w.ring0 + (IS_V ? (size_t)C::rsp0 * kPitchL : (size_t)C::SRC_RING_F2);
    w.ring2 = w.ring1 + (size_t)C::rsp1 * kPitchL;
    w.stage = w.ring2 + (size_t)C::rsp2 * kPitchL;
    w.mbar0 = 0;
    w.mpar = 0;
    if constexpr (C::MBAR) {
        // the warp's own barriers (behind its rings): every lane arrives once per group, either
        // with its cp.async copies (checked rounds) or plainly beside lane 0's bulk copies
        float2* bars = sm + (IS_V ? C::WARP_F2_V : C::WARP_F2_H) - C::MBAR_F2;
        w.mbar0 = smem_u32(bars);
#if defined(__CUDACC__)
        if (lane == 0) {
            for (int i = 0; i < C::NG; ++i) mbar_init(w.mbar0 + i * 8, 32);
            mbar_init_fence();
        }
        __syncwarp();
#endif
    }
    const int rho_first = p.out0 / C::B, rho_last = (p.out1 - 1) / C::B;
    const int rps = rho_last - rho_first + 1;
    const int nstrips = stream_strip_count(p);
    const long long units = (long long)nstrips * rps;
    long long u0 = gw * units / nwarps;
    const long long u1 = (gw + 1) * units / nwarps;
    while (u0 < u1) {
        const int strip = (int)(u0 / rps);
        const int r0 = (int)(u0 - (long long)strip * rps);
        const long long left = u1 - u0;
        const int rounds = (left < (long long)(rps - r0)) ? (int)left : rps - r0;
        run_warp<C, IS_V, EPI>(p, w, strip, rho_first + r0, rounds);
        u0 += rounds;
    }
}

#if defined(__CUDACC__)
template <class C, bool IS_V, int EPI>
__global__ void __launch_bounds__((IS_V ? C::NWARPS_V : C::NWARPS_H) * 32, 1)
stream_pass_kernel(const __grid_constant__ StreamParams p) {
    constexpr int NW = IS_V ? C::NWARPS_V : C::NWARPS_H;
    constexpr bool SRGB = !IS_V && (C::SRCT == kSrcU8Srgb);
    __shared__ float slut[SRGB ? 256 : 1];
    if constexpr (SRGB) {
        for (int i = threadIdx.x; i < 256; i += NW * 32) slut[i] = __ldg(p.srgb_lut + i);
        __syncthreads();
    }
    extern __shared__ __align__(128) unsigned char stream_smem[]; // (tensor copies land 128-byte aligned)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float2* sm = reinterpret_cast<float2*>(stream_smem) + (size_t)warp * (IS_V ? C::WARP_F2_V : C::WARP_F2_H);
    stream_warp_main<C, IS_V, EPI>(p, (long long)blockIdx.x * NW + warp, (long long)gridDim.x * NW, lane, sm, slut);
}
#endif

// ---- the chains ------------------------------------------------------------------------------------------
// (kind, summation, taps, advance) per step; final batches per round; source look-ahead in rounds.

// (scheduling variants and their defaults: stream_types.h)

// Source look-ahead in rounds (LAH row pass, LAV column pass) is what shared memory affords at
// 8 warps per SM: the row pass carries the staging rows, three-step chains a second
// intermediate ring.  RWU: rounds per trip of the register-window loop.  The source window of a
// chain closes on itself -- no register moves at the loop's back edge -- after WR0 / SRC_N rounds,
// rounded up, but three rounds of the headline chain are 31 KB of code and ran 34 % SLOWER than
// one round with its ~60 moves (profiles/r02a_sweep.jsonl: the instruction cache is a first-order
// effect here), so every chain runs one round per trip.  VAR = ChainC MODE.
#ifndef AVS_RWU_OVERRIDE
#define AVS_RWU_OVERRIDE 0
#endif
template <class S0, class S1, class S2, int REPS_LAST, int LAH, int LAV, int RWU, int VAR, bool IS_V, int SRCT, int NWMAX = 8>
using ChainV = ChainC<S0, S1, S2, REPS_LAST, (IS_V ? LAV : LAH), (VAR == 2 && !IS_V) ? 1 : VAR, IS_V ? AVIRB200_F32 : SRCT,
                      AVS_RWU_OVERRIDE ? AVS_RWU_OVERRIDE : RWU, NWMAX>;

// cfg3, float8_dil mirror (k = 2): RESIZE(24 taps, source step 2) -> 8-tap correction FIR
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainDil24 = ChainV<StepC<K_RESIZE, AVIRB200_SUM_DIL8, 24, 2>, StepC<K_FIR, AVIRB200_SUM_DIL8, 8, 1>, NoStep,
                          1, 2, 3, 1, VAR, IS_V, SRCT>;
// the same chain in 4-output batches: a 30-position window and half the code per round, small
// enough (<= 168 registers, <= 18.9 KB of rings) for THREE warps per scheduler
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainDil24Q = ChainV<StepC<K_RESIZE, AVIRB200_SUM_DIL8, 24, 2, 4>, StepC<K_FIR, AVIRB200_SUM_DIL8, 8, 1, 4>, NoStep,
                           1, 3, 3, 1, VAR, IS_V, SRCT, 12>;
// k = 2 in build mode 1, interleaved classes (fpclass_def<float>, fpclass_float4): RESIZE(24) -> FIR(7)
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainInl24 = ChainV<StepC<K_RESIZE, AVIRB200_SUM_INL, 24, 2>, StepC<K_FIR, AVIRB200_SUM_INL, 7, 1>, NoStep,
                          1, 2, 3, 1, VAR, IS_V, SRCT>;
// cfg3, float4 mirror (k = 2, build mode 0): FIR(7) -> RESIZE(18, source step 2) -> FIR(7)
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainInl3 = ChainV<StepC<K_FIR, AVIRB200_SUM_INL, 7, 1>, StepC<K_RESIZE, AVIRB200_SUM_INL, 18, 2>,
                         StepC<K_FIR, AVIRB200_SUM_INL, 7, 1>, 1, 1, 2, 1, VAR, IS_V, SRCT>;
// cfg4 (k = 4, build mode 0): FIR(15, decimation 2) -> RESIZE(18, source step 2) -> FIR(7)
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainInl3D = ChainV<StepC<K_FIR, AVIRB200_SUM_INL, 15, 2>, StepC<K_RESIZE, AVIRB200_SUM_INL, 18, 2>,
                          StepC<K_FIR, AVIRB200_SUM_INL, 7, 1>, 1, 1, 1, 1, VAR, IS_V, SRCT>;
// cfg5, float8_dil mirror (k = 4, build mode 1): RESIZE(56 taps, source step 4; 4-output batches) -> FIR(8)
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainDil56 = ChainV<StepC<K_RESIZE, AVIRB200_SUM_DIL8, 56, 4, 4>, StepC<K_FIR, AVIRB200_SUM_DIL8, 8, 1, 4>, NoStep,
                          1, 1, 1, 1, VAR, IS_V, SRCT>;
// cfg2 (k = 0.5): FIR(7) -> RESIZE(24) over the virtual 2X line; 32 final outputs per round
template <int VAR, bool IS_V, int SRCT = AVIRB200_F32>
using ChainUp2 = ChainV<StepC<K_FIR, AVIRB200_SUM_INL, 7, 1>, StepC<K_RESIZE2, AVIRB200_SUM_INL, 24, 1>, NoStep,
                        2, 1, 3, 1, VAR, IS_V, SRCT>;

template <class C>
struct ChainTag {
    using type = C;
};

template <bool V>
struct PassTag {
    static constexpr bool is_v = V;
};

// Calls f(ChainTag<Chain>(), PassTag<is_v>()) with the description of chain ID in scheduling
// variant `variant` for the row pass (is_v false) or the column pass.  Integer sources (row
// pass only) have two instantiations each: ring windows (variants 0, 3) and register windows.
// One chain per call so that every chain's kernels can live in their own translation unit
// (stream_chain.cu is compiled once per chain, in parallel).
template <int ID, class F>
inline bool stream_dispatch_chain(bool is_v, int variant, int src_type, F&& f) {
#define AVS_V(NAME, N)                                                                    \
    case N:                                                                               \
        if (is_v) f(ChainTag<NAME<N, true> >(), PassTag<true>());                         \
        else f(ChainTag<NAME<N, false> >(), PassTag<false>());                            \
        return true;
// (variant 3, every round on the checked path, exists in the host emulation only: it is the
// cross-check of the other variants' index logic, not something to launch)
#if defined(__CUDACC__)
#define AVS_V3(NAME)
#else
#define AVS_V3(NAME) AVS_V(NAME, 3)
#endif
#define AVS_INT_SRC(NAME, T)                                                              \
    if (!is_v && src_type == T) {                                                         \
        if (variant == 0 || variant == 3) f(ChainTag<NAME<0, false, T> >(), PassTag<false>()); \
        else f(ChainTag<NAME<1, false, T> >(), PassTag<false>());                         \
        return true;                                                                      \
    }
#define AVS_VARIANTS(NAME)                                                                \
    AVS_INT_SRC(NAME, AVIRB200_U8)                                                        \
    AVS_INT_SRC(NAME, AVIRB200_U16)                                                       \
    AVS_INT_SRC(NAME, kSrcU8Srgb)                                                         \
    switch (variant) {                                                                    \
        AVS_V(NAME, 0) AVS_V(NAME, 1) AVS_V(NAME, 2) AVS_V3(NAME)                         \
    default: return false;                                                                \
    }
    if (variant < 0 || variant >= kStreamVariants) return false;
    if constexpr (ID == kChainDil24) { AVS_VARIANTS(ChainDil24) }
    else if constexpr (ID == kChainInl24) { AVS_VARIANTS(ChainInl24) }
    else if constexpr (ID == kChainInl3) { AVS_VARIANTS(ChainInl3) }
    else if constexpr (ID == kChainInl3D) { AVS_VARIANTS(ChainInl3D) }
    else if constexpr (ID == kChainDil56) { AVS_VARIANTS(ChainDil56) }
    else if constexpr (ID == kChainUp2) { AVS_VARIANTS(ChainUp2) }
    else if constexpr (ID == kChainDil24Q) { AVS_VARIANTS(ChainDil24Q) }
    else return false;
#undef AVS_VARIANTS
#undef AVS_INT_SRC
#undef AVS_V3
#undef AVS_V
}

// The same for a run-time chain id (the host emulation: everything in one translation unit).
template <class F>
inline bool stream_dispatch(int id, bool is_v, int variant, int src_type, F&& f) {
    switch (id) {
    case kChainDil24: return stream_dispatch_chain<kChainDil24>(is_v, variant, src_type, f);
    case kChainInl24: return stream_dispatch_chain<kChainInl24>(is_v, variant, src_type, f);
    case kChainInl3: return stream_dispatch_chain<kChainInl3>(is_v, variant, src_type, f);
    case kChainInl3D: return stream_dispatch_chain<kChainInl3D>(is_v, variant, src_type, f);
    case kChainDil56: return stream_dispatch_chain<kChainDil56>(is_v, variant, src_type, f);
    case kChainUp2: return stream_dispatch_chain<kChainUp2>(is_v, variant, src_type, f);
    case kChainDil24Q: return stream_dispatch_chain<kChainDil24Q>(is_v, variant, src_type, f);
    default: return false;
    }
}

} // namespace avs
