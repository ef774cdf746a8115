/* avirb200.h -- C ABI of libavirb200.so, the H100 (sm_90a) execution engine behind the
 * header-only avir::CImageResizer<> / avir::CLancIR drop-in front-ends (avir_b200.h,
 * lancir_b200.h).
 *
 * Upstream AVIR has no FFI of its own (it is a header-only C++ template library), so this
 * boundary sits where a GPU can replace it: at the granularity of one
 * CImageResizer<>::resizeImage() call (upstream avir.h:4680-5092) resp. one
 * CLancIR::resizeImage() call (upstream lancir.h:386-713).  The host front-end does what
 * upstream does on the host -- decide the chain of filtering steps and design their
 * coefficients in double precision (upstream avir.h:5128-6270) -- and hands the result to
 * this library as a flat, pointer-and-size "plan descriptor".  The library owns only
 * device-side work: upload of the tables, the row pass, the column pass, the output
 * epilogue, and the inter-GPU halo exchange.
 *
 * Conventions: every function returns 0 on success or a negative avirb200_status; no
 * function throws; no function falls back to the CPU.  Plans are immutable after creation
 * and may be shared by threads/streams; a workspace belongs to one in-flight call.
 */
#ifndef AVIRB200_H
#define AVIRB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum avirb200_status {
    AVIRB200_OK = 0,
    AVIRB200_ERR_BAD_ARG = -1,
    AVIRB200_ERR_CUDA = -2,
    AVIRB200_ERR_NCCL = -3,
    AVIRB200_ERR_UNSUPPORTED = -4,
    AVIRB200_ERR_NO_DEVICE = -5,
    AVIRB200_ERR_ALLOC = -6
} avirb200_status;

/* Element types of the caller's image buffers (upstream Tin/Tout, avir.h:4670-4677).
 * F64: upstream narrows double input with a (float) cast in packScanline and widens the float
 * result with a (double) cast in unpackScanline (avir.h:2803-2806, 3168-3171); the library
 * does the same casts on the device, on every AVIR entry point (the sharded calls cast each
 * rank's own bands, the per-pass entry points cast in the row pass and in the column pass).
 * U32: LANCIR plans only (upstream lancir.h treats uint32_t as uint16_t): read as (float) v, no clamp on
 * input, output clamped to [0, 65535] and stored 32 bits wide.  AVIR plans take U8 / U16 / F32 / F64. */
typedef enum avirb200_dtype {
    AVIRB200_U8 = 0,
    AVIRB200_U16 = 1,
    AVIRB200_F32 = 2,
    AVIRB200_F64 = 3,
    AVIRB200_U32 = 4
} avirb200_dtype;

/* Step kinds of a 1-D filtering chain (upstream CImageResizerFilterStep, avir.h:2568-2728). */
typedef enum avirb200_step_kind {
    AVIRB200_STEP_FIR = 0,      /* doFilter  (avir.h:3748-3866, avir_dil.h:444-539) */
    AVIRB200_STEP_UPSAMPLE = 1, /* doUpsample with filtering (avir.h:3404-3733) */
    AVIRB200_STEP_RESIZE = 2    /* doResize / doResize2 (avir.h:3884-4328, avir_dil.h:559-761);
                                   a filterless 2X upsample in front of it is folded in */
} avirb200_step_kind;

/* Tap-accumulation order to mirror (this is what makes results bit-identical):
 *   INL  : upstream interleaved classes (fpclass_def<float>, fpclass_float4) -- sequential.
 *   DIL8 : upstream fpclass_float8_dil -- 8 lane-strided partial sums + float8::hadd tree
 *          (avir_dil.h:463-472,598-609; avir_float8_avx.h:264-273). */
typedef enum avirb200_sum_mode { AVIRB200_SUM_INL = 0, AVIRB200_SUM_DIL8 = 1 } avirb200_sum_mode;

/* Integer-output rounding to mirror (upstream CDitherer::dither + round()):
 *   HALFUP_INT : avir::round<float>, (int)(v+0.5) (avir.h:130-135)      -- fpclass_def<float>
 *   RNE_I32    : round(float4) through cvtps_epi32 (avir_float4_sse.h:303-313)
 *   RNE        : round(float8), _mm256_round_ps nearest-even (avir_float8_avx.h:347-351) */
typedef enum avirb200_round_mode {
    AVIRB200_ROUND_HALFUP_INT = 0,
    AVIRB200_ROUND_RNE_I32 = 1,
    AVIRB200_ROUND_RNE = 2
} avirb200_round_mode;

#define AVIRB200_MAX_STEPS 6

/* One filtering step.  All pointers are HOST pointers, copied by avirb200_plan_create. */
typedef struct avirb200_step_desc {
    int32_t kind;       /* avirb200_step_kind */
    int32_t resample;   /* FIR: decimation R >= 1; UPSAMPLE: factor (2) */
    int32_t latency;    /* FIR / UPSAMPLE: filter latency L */
    int32_t edge;       /* FIR: extra edge outputs per side (EdgePixelCount) */
    int32_t in_len;     /* input line length n; reads are clamped to [0, n-1] */
    int32_t out_len;    /* outputs produced */
    int32_t ntaps;      /* FIR/UPSAMPLE: taps stored; RESIZE: bank filter length FL */
    int32_t order;      /* RESIZE: 0 or 1 (c0 + c1*x) */
    int32_t upsampled;  /* RESIZE: input is the virtual 2X zero-stuffed line */
    int32_t skip_odd;   /* RESIZE: accumulate only taps that land on real samples (doResize2) */
    int32_t zero_start; /* accumulators start at +0 (avir.h:3938-3951, avir_dil.h:645) */
    int32_t nphases;    /* RESIZE: phases stored in taps[] */
    int32_t out_prefix; /* UPSAMPLE: outputs produced before position 0 */
    int32_t out_suffix; /* UPSAMPLE: outputs produced after position out_len-1 */
    int32_t in_prefix;  /* UPSAMPLE: times the first sample is additionally filtered */
    int32_t in_suffix;  /* UPSAMPLE: times the last sample is additionally filtered */
    int32_t n_prefix_dc, n_suffix_dc;
    const float* taps;       /* FIR/UPSAMPLE: ntaps; RESIZE: nphases*ntaps*(order+1) */
    const int32_t* src_pos;  /* RESIZE: out_len integer source positions (SrcPosInt) */
    const int32_t* phase;    /* RESIZE: out_len indices into taps[] phases */
    const float* frac;       /* RESIZE: out_len interpolation fractions x */
    const float* prefix_dc;  /* UPSAMPLE */
    const float* suffix_dc;  /* UPSAMPLE */
} avirb200_step_desc;

typedef struct avirb200_axis_desc {
    int32_t src_len, dst_len, nsteps;
    avirb200_step_desc steps[AVIRB200_MAX_STEPS];
} avirb200_axis_desc;

typedef struct avirb200_plan_desc {
    int32_t src_w, src_h, dst_w, dst_h;
    int32_t channels;        /* 1..4 (ElCountIO) */
    int32_t in_type, out_type; /* avirb200_dtype */
    int32_t sum_mode;        /* avirb200_sum_mode */
    int32_t round_mode;      /* avirb200_round_mode (integer output only) */
    int32_t use_gamma;       /* bit 0: sRGB-linearise the input; bit 1: de-linearise the output */
    int32_t alpha_index;     /* channel exempt from gamma when channels == 4 (0 or 3), else -1 */
    float in_gamma_mult;     /* (float)Vars.InGammaMult  (avir.h:2843) */
    float out_gamma_mult;    /* (float)Vars.OutGammaMult (avir.h:2987) */
    float tr_mul, tr_mul_inv; /* bit-depth truncation multipliers (avir.h:4408-4417); 1 = off */
    float pk_out;            /* output clamp ceiling (avir.h:5043) */
    int32_t dither;          /* integer output: 0 = per-sample rounding (CImageResizerDithererDefINL/DIL,
                                avir.h:4392-4419), 1 = error diffusion (CImageResizerDithererErrdINL/DIL,
                                avir.h:4442-4530, avir_dil.h:882-986): row-recursive; on the sharded calls
                                each band continues from the last row of the band above; not in windows */
    avirb200_axis_desc h, v; /* row pass, column pass */
} avirb200_plan_desc;

typedef struct avirb200_plan avirb200_plan; /* opaque, device-resident tables */

/* ---- single-GPU path --------------------------------------------------------------- */

/* Copies the descriptor's tables to the current CUDA device.
 * Every pass must fit the generic kernel with one output of one line per block: the source span of
 * that output (about 19 x the downscale ratio on the axis, at most the line) times (channels | 1)
 * floats, in the device's opt-in shared memory per block.  A plan that does not fit is refused here
 * with AVIRB200_ERR_UNSUPPORTED and a message naming the pass; no call of a created plan fails for
 * this reason.  On an H100 (227 KiB per block) this refuses only 4-channel lines of more than about
 * 11 600 source pixels resized to very few pixels (e.g. 16384 x 4 -> 1 x 4 RGBA). */
int avirb200_plan_create(const avirb200_plan_desc* desc, avirb200_plan** out);
void avirb200_plan_destroy(avirb200_plan* plan);

/* Bytes of device scratch one call needs (the fp32 row-pass intermediate,
 * upstream FltBuf, avir.h:4881-4883). */
int avirb200_plan_workspace_bytes(const avirb200_plan* plan, size_t* bytes);

/* Device-resident resize: src/dst/workspace are device pointers, pitches are in ELEMENTS
 * (upstream SrcScanlineSize semantics, avir.h:4647-4649).  Asynchronous on `stream`
 * (a cudaStream_t passed as void*); no allocation, no synchronisation. */
int avirb200_resize_device(const avirb200_plan* plan, const void* d_src, size_t src_pitch,
                           void* d_dst, size_t dst_pitch, void* d_workspace, void* stream);

/* The two passes of avirb200_resize_device individually (same arguments, same stream
 * semantics): row pass src -> workspace, column pass workspace -> dst.  For callers that
 * pipeline frames, and for per-kernel timing.  A double source is cast to floats in the workspace
 * by the row pass; the column pass of a double-output or error-diffusion plan writes float rows
 * into the workspace and then widens or dithers them (the workspace is avirb200_plan_workspace_bytes). */
int avirb200_row_pass_device(const avirb200_plan* plan, const void* d_src, size_t src_pitch,
                             void* d_workspace, void* stream);
int avirb200_col_pass_device(const avirb200_plan* plan, const void* d_workspace, void* d_dst,
                             size_t dst_pitch, void* stream);

/* HOST ENTRY POINTS (avirb200_resize_host, avirb200_resize_window_host, avirb200_resize_sharded_host and
 * CLancIR's lancirb200_resize_host, _window_host and _sharded_host) share one contract.  Pitches are in
 * elements; a pitch smaller than a row of the caller's image is AVIRB200_ERR_BAD_ARG before any CUDA call.
 * The call runs on the plan's device, whichever device is current, and the caller's current device is
 * unchanged afterwards.  It copies the caller's rows into device staging buffers, runs the device call on
 * the plan's own stream, copies the result out and synchronises.  AVIR plans stage in buffers shared by
 * every AVIR plan of the device, so AVIR host calls on one device run one at a time; a CLancIR plan stages
 * in buffers of its own.  Host calls on one plan run one at a time.  Pageable or page-locked memory. */

/* Convenience used by the drop-in resizeImage(): host buffers in, host buffers out
 * (H2D, both passes, D2H, synchronise).
 * Images of 64 MiB and more are cut into row bands travelling on separate copy-in / compute /
 * copy-out streams, so that the PCIe transfers of both directions overlap each other and the
 * kernels (page-locked host memory lets them run asynchronously); the result bits do not
 * depend on the banding.  h_dst may alias h_src (upstream allows NewBuf == SrcBuf when the
 * destination is not larger, avir.h:4650-4652): such calls run unbanded. */
int avirb200_resize_host(avirb200_plan* plan, const void* h_src, size_t src_pitch, void* h_dst,
                         size_t dst_pitch);

/* Number of kernel launches the last avirb200_resize_device on this plan issued.  Under concurrent
 * calls on one plan it is the count of one of those calls. */
int avirb200_plan_last_launches(const avirb200_plan* plan);

/* Video / batch entry: `n` frames of the plan's geometry, one launch pair per frame, all on
 * `stream` in order (the frames share `d_workspace`: stream order keeps them apart).  d_srcs /
 * d_dsts are HOST arrays of n device pointers; pitches as in avirb200_resize_device.  The
 * plan-building cost (host filter design, table upload) is paid once for the whole batch --
 * upstream's equivalent is re-using one CImageResizer object and its Vars across frames. */
int avirb200_resize_device_batch(const avirb200_plan* plan, int n, const void* const* d_srcs,
                                 size_t src_pitch, void* const* d_dsts, size_t dst_pitch,
                                 void* d_workspace, void* stream);

/* ---- destination windows ------------------------------------------------------------- */

/* A window is the destination sub-rectangle [x0, x0 + w) x [y0, y0 + h) of the plan's full
 * src_w x src_h -> dst_w x dst_h resize.  Its pixels are bit-identical to the same pixels of
 * avirb200_resize_device on the whole image, and a call reads only the window's source
 * footprint and filters only the intermediate the window needs.  Windows must be non-empty and
 * lie inside the destination (AVIRB200_ERR_BAD_ARG, before any CUDA call); plans with
 * error diffusion, whose every pixel depends on all pixels before it, return
 * AVIRB200_ERR_UNSUPPORTED. */
typedef struct avirb200_window_info {
    int32_t src_x0, src_w;      /* source columns the window reads (clamped to the image: reads */
    int32_t src_y0, src_h;      /*   past an edge replicate the edge), and source rows */
    int32_t mid_row0, mid_rows; /* intermediate rows the column pass reads (= the source rows) */
} avirb200_window_info;

/* The footprint of a window.  Also builds the tile kernel's device tables of the window's column and
 * row ranges (once per window: an allocation and a synchronous copy; avirb200_window_workspace_bytes
 * does the same).  A window queried first runs its passes on the tile kernel where the plan has it; a
 * window never queried runs them on the generic kernel, with the same bits (a 1920 x 1080 window of
 * 7680 x 4320 -> 5120 x 2880 RGBA u8 took 4.2 x as long on an H100 80GB HBM3 at 700 W:
 * profiles/h100_streams.txt).  avirb200_resize_window_device never builds a table: it stays
 * asynchronous, allocation-free and capturable into a CUDA graph either way. */
int avirb200_window_query(const avirb200_plan* plan, int x0, int y0, int w, int h, avirb200_window_info* info);
/* Same, from a descriptor alone (pure host arithmetic, no device needed). */
int avirb200_window_query_desc(const avirb200_plan_desc* desc, int x0, int y0, int w, int h,
                               avirb200_window_info* info);
/* Workspace of one window call: the intermediate (mid_rows x w pixels of floats) and, where the
 * plan uses them, the float copies of double buffers and the 4-channel copies of 1..3-channel
 * images, sized for the footprint and the window. */
int avirb200_window_workspace_bytes(const avirb200_plan* plan, int x0, int y0, int w, int h, size_t* bytes);
/* d_src points at the footprint's first pixel (source pixel (src_x0, src_y0)) and holds the
 * footprint's src_w x src_h pixels; d_dst points at the window's first pixel and receives w x h
 * pixels.  Pitches in elements, as in avirb200_resize_device; the same stream rules (no
 * allocation, no synchronisation). */
int avirb200_resize_window_device(const avirb200_plan* plan, int x0, int y0, int w, int h, const void* d_src,
                                  size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_workspace,
                                  void* stream);
/* The same with HOST buffers (a host entry point): h_src is the WHOLE source image (only the footprint is
 * copied to the device), h_dst receives the w x h window. */
int avirb200_resize_window_host(avirb200_plan* plan, int x0, int y0, int w, int h, const void* h_src,
                                size_t src_pitch, void* h_dst, size_t dst_pitch);

/* Per-plan options (tuning and test switches; none changes a result bit).  Options are plan
 * state: set them while no call on the plan is in flight.  value < 0 restores the default. */
typedef enum avirb200_option {
    /* kernel family order: 0 = streaming kernel where the chain is regular, else the tile kernel,
     * else the generic kernel (default); 1 = generic kernel only; 2 = tile kernel, else generic */
    AVIRB200_OPT_KERNEL_FAMILY = 0,
    /* scheduling variant of the streaming row / column pass: 0 ring windows, 1 register windows,
     * 2 register windows + TMA-staged source ring (column pass) */
    AVIRB200_OPT_STREAM_VARIANT_H = 1,
    AVIRB200_OPT_STREAM_VARIANT_V = 2,
    /* avirb200_resize_host: number of row bands of the pipelined form (1 = unbanded; default by size) */
    AVIRB200_OPT_HOST_BANDS = 3,
    /* 1: also select the streaming chains that measured slower than the tile kernel (upsizing, 56-tap) */
    AVIRB200_OPT_ALL_STREAM_CHAINS = 4,
    /* avirb200_resize_sharded, how the halo rows travel.  3 (default) = the FUSED exchange: the row
     * kernel itself stores the rows the neighbours need into their mailboxes (peer stores over NVLink)
     * and raises their flags, the column kernel reads the neighbours' rows in place from the mailbox --
     * no exchange stream, no copies, no extra launch (a pass that is not on the streaming kernel falls
     * back to the push / pull of 1, per pass).  1 = rows pushed by the copy engines into the
     * neighbours' mailboxes after the row pass, pulled into the workspace by a small kernel; 2 = the
     * same with the rows the neighbours need filtered FIRST (one segmented launch) so that the push
     * overlaps the interior rows; 0 = NCCL send/recv between the two passes. */
    AVIRB200_OPT_OVERLAP_HALO = 5
} avirb200_option;
int avirb200_plan_set_option(avirb200_plan* plan, int option, int value);

/* ---- row-sharded multi-GPU path (one process per GPU) -------------------------------- */

/* Source/destination row ranges rank `rank` of `nranks` owns, and the intermediate rows it
 * must receive from its neighbours before the column pass (SURVEY.md section 8e). */
typedef struct avirb200_shard_info {
    int32_t src_row0, src_rows; /* source rows this rank filters in the row pass */
    int32_t dst_row0, dst_rows; /* destination rows this rank produces */
    int32_t need_row0, need_rows; /* intermediate rows the column pass reads */
    int32_t halo_up, halo_down;   /* rows received from rank-1 / rank+1 */
} avirb200_shard_info;

int avirb200_shard_query(const avirb200_plan* plan, int rank, int nranks,
                         avirb200_shard_info* info);
/* Same, from a descriptor alone (pure host arithmetic, no device needed). */
int avirb200_shard_query_desc(const avirb200_plan_desc* desc, int rank, int nranks,
                              avirb200_shard_info* info);
int avirb200_shard_workspace_bytes(const avirb200_plan* plan, int rank, int nranks,
                                   size_t* bytes);
/* From a descriptor alone (pure host arithmetic, no device needed): the rank's
 * avirb200_shard_workspace_bytes and the bytes of its halo mailbox (header and both call-parity
 * slots: the halo rows from above and below and, with error diffusion, the ditherer's row from the
 * rank above; the allocation is rounded up to 2 MiB).  Only for plans whose passes keep the image's
 * channel count -- 4 channels, double buffers or error diffusion; a 1..3-channel plan of another kind
 * may run widened to 4 channels, which plan creation decides: AVIRB200_ERR_UNSUPPORTED. */
int avirb200_shard_layout_desc(const avirb200_plan_desc* desc, int rank, int nranks, size_t* ws_bytes,
                               size_t* mailbox_bytes);

/* NCCL bootstrap without exposing NCCL types: rank 0 fills a 128-byte id, the caller
 * broadcasts it by any means, every rank then creates its communicator. */
int avirb200_comm_unique_id(void* id128);
int avirb200_comm_create(const void* id128, int rank, int nranks, void** comm_out);
void avirb200_comm_destroy(void* comm);

/* d_src holds this rank's source band (src_rows rows), d_dst receives its destination band
 * (dst_rows rows).  Row pass -> NCCL halo send/recv with rank-1/rank+1 -> column pass, all
 * enqueued on `stream`.  `comm` is an ncclComm_t (from avirb200_comm_create or the
 * caller's own).  Output is bit-identical to the single-GPU path.
 * Default schedule (AVIRB200_OPT_OVERLAP_HALO = 3): every rank owns a mailbox in device memory that its
 * neighbours map through CUDA IPC (the handles travel over `comm` once per plan).  The row kernel
 * stores the rows a neighbour needs into that neighbour's mailbox as it produces them and, when the
 * last one is out, the call's sequence number into the neighbour's flag; the column kernel reads
 * the neighbours' rows in place from its own mailbox, and only the runs that touch them wait for
 * the flag.  The first call on a plan is collective (every rank must make it).  Where peer mapping
 * is unavailable the NCCL send/recv schedule runs.
 * Double buffers: each rank casts its own source band to floats and its float result to doubles.
 * Error diffusion: each rank dithers its own rows, starting from the D row the rank above left; that
 * row travels through the rank's mailbox (peer stores and a progress word naming the call) or, on the
 * NCCL schedule and below a rank that reads no rows from the rank under it, with ncclSend / ncclRecv
 * after the rank above has dithered.  The ditherer is a wavefront through the whole image: its time does not
 * shrink with more ranks, only the passes' does. */
int avirb200_resize_sharded(const avirb200_plan* plan, void* comm, int rank, int nranks,
                            const void* d_src, size_t src_pitch, void* d_dst, size_t dst_pitch,
                            void* d_workspace, void* stream);

/* The same with HOST buffers (a host entry point): this rank's source band in, its destination band
 * out, through avirb200_resize_sharded on the plan's own stream.  The multi-GPU form of
 * avirb200_resize_host. */
int avirb200_resize_sharded_host(avirb200_plan* plan, void* comm, int rank, int nranks,
                                 const void* h_src, size_t src_pitch, void* h_dst, size_t dst_pitch);

/* Validation aid: runs the `nranks` bands of the sharded schedule one after another on the
 * CURRENT device.  With the default AVIRB200_OPT_OVERLAP_HALO (3) the bands exchange their halo rows
 * exactly as ranks do -- the row kernel stores them into the neighbour band's mailbox (here in local
 * memory) and raises its flag, the column kernel reads them in place; otherwise with device copies.
 * Error diffusion hands each band's last D row to the next band through the same kind of mailbox.
 * Full-image device buffers; d_workspace must hold the sum of all ranks'
 * avirb200_shard_workspace_bytes. */
int avirb200_resize_sharded_local(const avirb200_plan* plan, int nranks, const void* d_src,
                                  size_t src_pitch, void* d_dst, size_t dst_pitch,
                                  void* d_workspace, void* stream);

/* Which specialised kernels the plan's passes qualify for: bit 0 / 1 = row / column pass on
 * the warp-streaming kernel, bit 2 / 3 = row / column pass on the tile kernel. */
int avirb200_plan_kernel_paths(const avirb200_plan* plan);

/* ---- LANCIR (upstream lancir.h) ------------------------------------------------------- */

typedef struct lancirb200_axis_desc {
    int32_t src_len, dst_len;
    int32_t kernel_len;     /* KernelLen (lancir.h:889-895) */
    int32_t nphases;
    const float* taps;      /* nphases * kernel_len, un-replicated (lancir.h:1076-1156) */
    const int32_t* src_pos; /* dst_len: first tap's source index (may be < 0 / >= src_len) */
    const int32_t* phase;   /* dst_len */
} lancirb200_axis_desc;

typedef struct lancirb200_plan_desc {
    int32_t src_w, src_h, dst_w, dst_h, channels;
    int32_t in_type, out_type; /* avirb200_dtype: U8, U16, F32, F64 or U32 */
    float out_mul;          /* lancir.h:526-533 */
    int32_t is_unity_mul;
    float clamp_max;        /* 255 / 65535 for integer output */
    lancirb200_axis_desc v, h; /* LANCIR resizes columns first, then rows */
} lancirb200_plan_desc;

typedef struct lancirb200_plan lancirb200_plan;

/* Element types, as upstream's CLancIR (lancir.h:373-381): the kernels read and write every type
 * natively.  Input: (float) v, rounded to nearest-even (F64 values beyond float's range become +-Inf,
 * float subnormals stay subnormal; U32 is exact up to 2^24 and not clamped).  F64 output: (double) of
 * the float result (times out_mul unless is_unity_mul), no clamp.  U32 output: as U16 -- clamped to
 * [0, clamp_max], nearest-even, the last (dst_w * channels) & 3 elements of a row (int)(v + 0.5f) --
 * stored 32 bits wide; a NaN in that tail stores x86's (int)NaN, 2147483648, as upstream does.  A type
 * code outside 0..4 is AVIRB200_ERR_BAD_ARG, before any CUDA call. */
int lancirb200_plan_create(const lancirb200_plan_desc* desc, lancirb200_plan** out);
void lancirb200_plan_destroy(lancirb200_plan* plan);
int lancirb200_plan_workspace_bytes(const lancirb200_plan* plan, size_t* bytes);
int lancirb200_resize_device(const lancirb200_plan* plan, const void* d_src, size_t src_pitch,
                             void* d_dst, size_t dst_pitch, void* d_workspace, void* stream);
/* Host buffers in and out (a host entry point, see avirb200_resize_host). */
int lancirb200_resize_host(lancirb200_plan* plan, const void* h_src, size_t src_pitch,
                           void* h_dst, size_t dst_pitch);

/* Destination windows of a LANCIR plan, as avirb200_*window* for AVIR: the window
 * [x0, x0 + w) x [y0, y0 + h) of the plan's full resize, bit-identical to the same pixels of
 * lancirb200_resize_device.  The column pass runs over the footprint's columns and the window's rows
 * only, the row pass over the window's columns only.  Windows must be non-empty and lie inside the
 * destination (AVIRB200_ERR_BAD_ARG, before any CUDA call); a window may be at most 65535 rows tall,
 * whatever the plan's height. */
typedef struct lancirb200_window_info {
    int32_t src_x0, src_w;   /* source columns the window reads, clamped to the image (reads past an */
    int32_t src_y0, src_h;   /*   edge replicate the edge), and source rows */
} lancirb200_window_info;

/* The footprint: every tap position of every window output, clamped to the image, min / max per axis
 * (zero-valued taps included).  Pure host arithmetic on the plan's own copy of the tables. */
int lancirb200_window_query(const lancirb200_plan* plan, int x0, int y0, int w, int h, lancirb200_window_info* info);
/* Same, from a descriptor alone (no device needed). */
int lancirb200_window_query_desc(const lancirb200_plan_desc* desc, int x0, int y0, int w, int h,
                                 lancirb200_window_info* info);
/* Workspace of one window call: the intermediate, h x src_w(footprint) pixels of floats. */
int lancirb200_window_workspace_bytes(const lancirb200_plan* plan, int x0, int y0, int w, int h, size_t* bytes);
/* d_src points at the footprint's first pixel (source pixel (src_x0, src_y0)) and holds its
 * src_w x src_h pixels; d_dst points at the window's first pixel and receives w x h pixels.  Pitches in
 * elements; asynchronous on `stream`, no allocation. */
int lancirb200_resize_window_device(const lancirb200_plan* plan, int x0, int y0, int w, int h, const void* d_src,
                                    size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_workspace,
                                    void* stream);
/* The same with HOST buffers (a host entry point, see avirb200_resize_host): h_src is the WHOLE source
 * image (only the footprint is copied to the device), h_dst receives the w x h window. */
int lancirb200_resize_window_host(lancirb200_plan* plan, int x0, int y0, int w, int h, const void* h_src,
                                  size_t src_pitch, void* h_dst, size_t dst_pitch);

/* Row-sharded LANCIR (one process per GPU), as avirb200_*sharded* for AVIR: rank r of n holds source rows
 * [src_h * r / n, src_h * (r + 1) / n) and produces destination rows [dst_h * r / n, dst_h * (r + 1) / n),
 * bit-identical to the same rows of lancirb200_resize_device.  LANCIR resizes columns first, so only raw
 * source rows travel between neighbours, in the caller's element type.  In avirb200_shard_info, need_row0 /
 * need_rows are SOURCE rows: the band's vertical footprint (every tap position of its destination rows,
 * clamped to the image, as lancirb200_window_query) joined with its own source band; halo_up / halo_down are
 * the source rows of it held by rank-1 / rank+1.  AVIRB200_ERR_UNSUPPORTED, before any CUDA call, when a
 * rank gets no rows, a halo is larger than the neighbour's band (too many ranks), or a band has more than
 * 65535 destination rows (a plan taller than that runs sharded when every band fits). */
int lancirb200_shard_query(const lancirb200_plan* plan, int rank, int nranks, avirb200_shard_info* info);
/* Same, from a descriptor alone (no device needed). */
int lancirb200_shard_query_desc(const lancirb200_plan_desc* desc, int rank, int nranks, avirb200_shard_info* info);
/* The band's intermediate (dst_rows x src_w x channels floats), the two halo segments the NCCL schedule
 * receives into and a 256-byte header. */
int lancirb200_shard_workspace_bytes(const lancirb200_plan* plan, int rank, int nranks, size_t* bytes);
/* d_src holds this rank's source band, d_dst receives its destination band; pitches in elements, at least a
 * row.  `comm` is an ncclComm_t (avirb200_comm_create or the caller's own); nranks == 1 is
 * lancirb200_resize_device.  The current device must be the plan's.  Asynchronous on `stream`; no allocation
 * after the first call on a plan, which is collective (every rank makes it): every rank allocates a mailbox
 * in device memory that its neighbours map through CUDA IPC (the handles travel over `comm`).  Per call a
 * rank copies the rows each neighbour needs into that neighbour's mailbox on an exchange stream forked from
 * `stream` (peer copies, no kernel of the call before them), then the call's sequence number into its flag;
 * the column pass reads the neighbours' rows in place, and only its blocks whose taps reach them wait for
 * the flag.  `stream` joins the exchange before the call returns.  A pair of neighbours where rows travel
 * one way only, and every pair when some rank cannot map its neighbours or AVIRB200_OPT_OVERLAP_HALO is 0,
 * exchanges with ncclSend / ncclRecv into the workspace's halo segments before the column pass. */
int lancirb200_resize_sharded(const lancirb200_plan* plan, void* comm, int rank, int nranks, const void* d_src,
                              size_t src_pitch, void* d_dst, size_t dst_pitch, void* d_workspace, void* stream);
/* The same with HOST buffers (a host entry point, see avirb200_resize_host): this rank's source band in,
 * its destination band out. */
int lancirb200_resize_sharded_host(lancirb200_plan* plan, void* comm, int rank, int nranks, const void* h_src,
                                   size_t src_pitch, void* h_dst, size_t dst_pitch);
/* Validation aid: every band of an `nranks` split on the CURRENT device, with full-image buffers.  The bands
 * exchange through mailboxes in their own workspaces with the same push, segmented column kernel and flag
 * protocol as ranks (AVIRB200_OPT_OVERLAP_HALO 0: device copies into the same segments, no waiting).
 * d_workspace holds the sum of every rank's lancirb200_shard_workspace_bytes, band after band. */
int lancirb200_resize_sharded_local(const lancirb200_plan* plan, int nranks, const void* d_src, size_t src_pitch,
                                    void* d_dst, size_t dst_pitch, void* d_workspace, void* stream);
/* CLancIR plans take one option, AVIRB200_OPT_OVERLAP_HALO: 3 (default, mailboxes) or 0 (every halo row
 * through NCCL on lancirb200_resize_sharded, device copies on _local).  A test switch: results do not change
 * by a bit.  Anything else is AVIRB200_ERR_BAD_ARG. */
int lancirb200_plan_set_option(lancirb200_plan* plan, int option, int value);

/* ---- misc ----------------------------------------------------------------------------- */

const char* avirb200_status_string(int status);
const char* avirb200_last_error(void); /* thread-local detail of the last failure */
int avirb200_device_count(void);

/* Self-test on the current device: the batched, branch-free output gamma of the streaming column pass
 * (pixel_ops.cuh, lin2srgb_batch: the library square root's fast path spelled out so that several
 * samples' chains interleave) against the one-sample path (upstream avir.h:288-310 evaluated with
 * sqrt.rn.f64) on EVERY float bit pattern the batched path accepts.  *checked = patterns compared,
 * *mismatches = patterns whose results differ in any bit (must be 0). */
int avirb200_selftest_lin2srgb(unsigned long long* checked, unsigned long long* mismatches);

#ifdef __cplusplus
}
#endif

#endif /* AVIRB200_H */
