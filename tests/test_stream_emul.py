"""Index logic of the warp-streaming pass kernel, checked WITHOUT a GPU: the kernel source
(avir_b200/csrc/stream_kernel.cuh) compiled for the host and executed in lockstep
(tests/emul/stream_emul.cpp: 32 threads per warp meeting at every __syncwarp) against the
oracle's C port executing the same plan descriptor.  Covers what differs from the tile
kernel: per-warp rings and pipeline delays, run splitting over warps, batches at the ends
of a line, ragged strips, destination bands of the sharded schedule.  The arithmetic itself
is shared with the device build; the GPU parity tests (-m gpu) cover the real kernel."""
import ctypes as C
import os

import numpy as np
import pytest

import cases as cs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
u8, u16, f32 = np.uint8, np.uint16, np.float32


class _SI(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_row0", "src_rows", "dst_row0", "dst_rows",
                                          "need_row0", "need_rows", "halo_up", "halo_down")]


def band_needs(dp, bands):
    """(need_row0, need_rows) of every band of the sharded schedule, or None where the product
    refuses the split (bands too small): the emulation then runs over the whole intermediate."""
    import avir_b200 as ab
    out = (C.c_int * (2 * bands))()
    for b in range(bands):
        si = _SI()
        if ab.lib().avirb200_shard_query_desc(C.c_void_p(dp), b, bands, C.byref(si)) != 0:
            return None
        out[2 * b], out[2 * b + 1] = si.need_row0, si.need_rows
    return out


def band_infos(dp, bands):
    """avirb200_shard_info of every band (8 ints each), or None where the product refuses the split."""
    import avir_b200 as ab
    out = (C.c_int * (8 * bands))()
    for b in range(bands):
        si = _SI()
        if ab.lib().avirb200_shard_query_desc(C.c_void_p(dp), b, bands, C.byref(si)) != 0:
            return None
        for i, (n, _) in enumerate(_SI._fields_):
            out[8 * b + i] = getattr(si, n)
    return out


@pytest.fixture(scope="module")
def emul():
    from avir_b200 import build as b
    lib = C.CDLL(b.build_emul())
    lib.stream_emul_resize.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                       C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    lib.stream_emul_resize.restype = C.c_int
    lib.stream_emul_resize_fused.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                             C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    lib.stream_emul_resize_fused.restype = C.c_int
    lib.stream_emul_applicable.argtypes = [C.c_void_p]
    lib.stream_emul_applicable.restype = C.c_int
    return lib


# (case, emulated warps of the row pass, of the column pass, destination bands)
EMUL_CASES = [
    ((2, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1}), 3, 2, 1),   # cfg3 chain, scaled down
    ((2, 192, 108, 96, 54, 4, f32, f32, 16, {}), 1, 1, 1),
    ((2, 384, 216, 192, 108, 4, f32, f32, 16, {}), 7, 5, 3),             # runs split inside strips
    ((2, 100, 70, 50, 35, 4, f32, f32, 16, {"buildmode": 1}), 4, 3, 2),   # ragged strips and batches
    ((2, 100, 70, 50, 35, 4, f32, u8, 8, {"buildmode": 1}), 4, 3, 2),     # integer output stage
    ((2, 100, 70, 50, 35, 4, f32, u16, 16, {"buildmode": 1}), 2, 2, 1),
    ((2, 20, 18, 10, 9, 4, f32, f32, 16, {"buildmode": 1}), 2, 2, 2),     # shorter than the pipeline
    ((2, 34, 6, 17, 3, 4, f32, f32, 16, {"buildmode": 1}), 1, 40, 1),     # more warps than rounds
    ((2, 640, 40, 320, 20, 4, f32, f32, 16, {"buildmode": 1}), 9, 2, 5),
    # interleaved classes, k = 2 in build mode 1: RESIZE(24) -> FIR(7)
    ((1, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1}), 3, 2, 1),
    ((0, 100, 70, 50, 35, 4, f32, u8, 8, {"buildmode": 1}), 4, 3, 2),
    ((1, 100, 70, 50, 35, 4, f32, u16, 16, {"buildmode": 1}), 2, 5, 3),
    # cfg3 float4 mirror chain (build mode 0): FIR(7) -> RESIZE(18) -> FIR(7)
    ((1, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 0}), 3, 2, 1),
    ((1, 100, 70, 50, 35, 4, f32, f32, 16, {"buildmode": 0}), 4, 3, 2),
    ((1, 20, 18, 10, 9, 4, f32, u8, 16, {"buildmode": 0}), 2, 2, 2),
    ((1, 640, 40, 320, 20, 4, f32, f32, 16, {"buildmode": 0}), 9, 2, 5),
    # cfg2 chain (k = 0.5, build mode 1): FIR(7) -> RESIZE(24) over the virtual 2X line
    ((1, 96, 54, 192, 108, 4, f32, f32, 8, {"buildmode": 1}), 3, 2, 1),
    ((1, 50, 35, 100, 70, 4, f32, u8, 8, {"buildmode": 1}), 4, 3, 2),
    ((1, 10, 9, 20, 18, 4, f32, f32, 8, {"buildmode": 1}), 2, 2, 2),
    ((1, 320, 20, 640, 40, 4, f32, u8, 8, {"buildmode": 1}), 9, 2, 5),
    # integer sources: raw pixels in the row pass's source ring, cast in the lanes' reads
    ((1, 96, 54, 192, 108, 4, u8, u8, 8, {"buildmode": 1}), 3, 2, 1),      # cfg2 as quoted (u8 -> u8)
    ((1, 50, 35, 100, 70, 4, u8, u8, 8, {"buildmode": 1}), 4, 3, 2),
    ((1, 10, 9, 20, 18, 4, u16, u16, 16, {"buildmode": 1}), 2, 2, 2),
    ((2, 192, 108, 96, 54, 4, u8, u8, 8, {"buildmode": 1}), 3, 2, 1),
    ((2, 100, 70, 50, 35, 4, u16, u16, 16, {"buildmode": 1}), 4, 3, 2),
    ((1, 100, 70, 50, 35, 4, u16, f32, 16, {"buildmode": 1}), 2, 5, 3),
    ((1, 100, 70, 50, 35, 4, u8, u8, 8, {"buildmode": 0}), 4, 3, 2),
    ((1, 640, 40, 320, 20, 4, u16, u16, 16, {"buildmode": 0}), 9, 2, 5),
    ((0, 20, 18, 10, 9, 4, u8, u16, 16, {"buildmode": 1}), 2, 2, 2),
    # cfg4 chain (k = 4, build mode 0): FIR(15, decimation 2) -> RESIZE(18) -> FIR(7)
    ((1, 384, 216, 96, 54, 4, u16, u16, 16, {"buildmode": 0}), 3, 2, 1),
    ((1, 200, 140, 50, 35, 4, u16, u16, 16, {"buildmode": 0}), 4, 3, 2),
    ((1, 200, 140, 50, 35, 4, f32, f32, 16, {"buildmode": 0}), 2, 5, 3),
    ((0, 40, 36, 10, 9, 4, u8, u8, 16, {"buildmode": 0}), 2, 2, 2),
    ((1, 1280, 80, 320, 20, 4, u16, u16, 16, {"buildmode": 0}), 9, 2, 5),
    # cfg5 chain (k = 4, build mode 1, float8_dil): RESIZE(56, step 4) in 4-output batches -> FIR(8);
    # u8 source linearised through the sRGB table in the lanes' reads, alpha exempt
    ((2, 384, 216, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3, "buildmode": 1}), 3, 2, 1),
    ((2, 200, 140, 50, 35, 4, u8, u8, 8, {"gamma": True, "alpha": 0, "buildmode": 1}), 4, 3, 2),
    ((2, 200, 140, 50, 35, 4, f32, f32, 16, {"buildmode": 1}), 2, 5, 3),
    ((2, 40, 36, 10, 9, 4, u8, u16, 16, {"gamma": True, "buildmode": 1}), 2, 2, 2),
    ((2, 1280, 80, 320, 20, 4, u16, u16, 16, {"buildmode": 1}), 9, 2, 5),
    ((2, 192, 108, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3, "buildmode": 1}), 3, 2, 1),  # k = 2 + sRGB source
]


def _id(ec):
    return "%s-w%d-%d-b%d" % (cs.case_id(ec[0]), ec[1], ec[2], ec[3])


# scheduling variants of the chain kernels (later steps' windows read ahead or not, separate
# straight-line loop for the interior rounds or not): all must produce the same bits
@pytest.mark.parametrize("variant", range(4))
@pytest.mark.parametrize("ec", EMUL_CASES, ids=_id)
def test_stream_kernel_emulation_matches_port(emul, ec, variant):
    case, wh, wv, bands = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        assert emul.stream_emul_applicable(dp) == 1, "chain not on the streaming kernel: %r" % (modes,)
        got = np.zeros((nh, nw, ch), to)
        lut = np.zeros(256, np.float32)
        cs.port().avir_port_srgb_lut(lut.ctypes.data)
        assert emul.stream_emul_resize(dp, src.ctypes.data, sw * ch, got.ctypes.data, nw * ch, wh, wv, bands,
                                       variant, lut.ctypes.data, 1, band_needs(dp, bands), (3 * variant + wh) % 23, (5 * variant + wv) % 19) == 0
    finally:
        rs.free_descriptor(h)
    want, _ = cs.port_output(case, src)
    assert cs.count_mismatch(want, got) == 0


# The sharded schedule with the fused halo exchange (AVIRB200_OPT_OVERLAP_HALO = 3): row passes store the
# boundary rows into the neighbours' mailboxes and raise their flags, column passes read them in place.
FUSED_CASES = [(ec[0], ec[1], ec[2], b) for ec in EMUL_CASES[::2] for b in (2, 3, 4)] + [
    # tall narrow images: middle bands with two neighbours, several strips between their rows
    ((2, 64, 400, 32, 200, 4, f32, f32, 16, {"buildmode": 1}), 3, 4, 3),
    ((2, 64, 400, 32, 200, 4, f32, f32, 16, {"buildmode": 1}), 5, 2, 4),
    ((1, 64, 400, 32, 200, 4, u16, u16, 16, {"buildmode": 0}), 2, 3, 4),
    ((2, 96, 640, 24, 160, 4, u8, u8, 8, {"gamma": True, "alpha": 3, "buildmode": 1}), 3, 2, 3),
    ((1, 48, 200, 96, 400, 4, u8, u8, 8, {"buildmode": 1}), 2, 3, 3),
    ((1, 128, 640, 32, 160, 4, u16, u16, 16, {"buildmode": 0}), 4, 3, 4),
]


@pytest.mark.parametrize("variant", (0, 1, 2))
@pytest.mark.parametrize("ec", FUSED_CASES, ids=_id)
def test_stream_kernel_emulation_fused_exchange_matches_port(emul, ec, variant):
    case, wh, wv, bands = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        infos = band_infos(dp, bands)
        if infos is None:
            pytest.skip("bands too small for the sharded schedule")
        got = np.zeros((nh, nw, ch), to)
        lut = np.zeros(256, np.float32)
        cs.port().avir_port_srgb_lut(lut.ctypes.data)
        rc = emul.stream_emul_resize_fused(dp, src.ctypes.data, sw * ch, got.ctypes.data, nw * ch, wh, wv, bands,
                                           variant, lut.ctypes.data, 1, infos)
        if rc == 1:
            pytest.skip("a strip with rows of both neighbours: the product pushes with the copy engines")
        assert rc == 0
    finally:
        rs.free_descriptor(h)
    want, _ = cs.port_output(case, src)
    assert cs.count_mismatch(want, got) == 0


# the headline chain's 4-output-batch twin (sweeps of 8 source positions, 12 warps per block on the device)
@pytest.mark.parametrize("variant", range(4))
@pytest.mark.parametrize("ec", [e for e in EMUL_CASES if e[0][0] == 2 and e[0][9].get("buildmode") == 1
                                and e[0][2] == 2 * e[0][4] and not e[0][9].get("gamma")], ids=_id)
def test_stream_kernel_emulation_q_chain_matches_port(emul, ec, variant):
    case, wh, wv, bands = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        out = (C.c_int * 4)()
        emul.stream_emul_selection.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        emul.stream_emul_selection(dp, 2, out)
        assert (out[0], out[1]) == (7, 7), list(out)
        got = np.zeros((nh, nw, ch), to)
        lut = np.zeros(256, np.float32)
        assert emul.stream_emul_resize(dp, src.ctypes.data, sw * ch, got.ctypes.data, nw * ch, wh, wv, bands,
                                       variant, lut.ctypes.data, 2, band_needs(dp, bands), wh % 7, 17 * (variant & 1)) == 0
    finally:
        rs.free_descriptor(h)
    want, _ = cs.port_output(case, src)
    assert cs.count_mismatch(want, got) == 0


def test_converted_sources_stay_on_the_tile_kernel(emul):
    # float / u16 input gamma is a double-precision polynomial per sample: not done in the lanes' reads
    case = (2, 100, 70, 50, 35, 4, f32, u16, 16, {"buildmode": 1, "gamma": True, "alpha": 3})
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor((70, 100, 4), f32, 50, 35, u16, 0.0, v)
    try:
        assert emul.stream_emul_applicable(dp) == 0
    finally:
        rs.free_descriptor(h)


def test_irregular_chains_stay_on_the_tile_kernel(emul):
    # non-integer ratio: positions are irregular and phases vary -> not a streaming chain
    case = (2, 150, 90, 100, 55, 4, f32, f32, 16, {"buildmode": 1})
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor((90, 150, 4), f32, 100, 55, f32, 0.0, v)
    try:
        assert emul.stream_emul_applicable(dp) == 0
    finally:
        rs.free_descriptor(h)


def test_chain_selection_of_the_baseline_configs(emul):
    """Which kernel family each BASELINE config's passes select (host logic shared with the
    engine): streaming chain ids per stream_types.h, 0 = tile kernel."""
    emul.stream_emul_selection.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    DIL24, INL24, INL3, INL3D, DIL56, UP2 = 1, 2, 3, 4, 5, 6
    U8, U16, F32, SRGB = 0, 1, 2, 4
    table = [
        # case (full BASELINE sizes; planning only)                                 default      all chains   src   epi
        ((1, 1920, 1080, 3840, 2160, 4, u8, u8, 8, {}),                             (UP2, 0),    (UP2, UP2),   U8,   2),   # cfg2: streaming row pass, tile column pass
        ((2, 7680, 4320, 3840, 2160, 4, f32, f32, 16, {}),                          (DIL24,) * 2, (DIL24,) * 2, F32, 1),   # cfg3
        ((1, 7680, 4320, 3840, 2160, 4, f32, f32, 16, {}),                          (INL3,) * 2, (INL3,) * 2,  F32,  1),
        ((1, 16384, 16384, 4096, 4096, 4, u16, u16, 16, {}),                        (INL3D,) * 2, (INL3D,) * 2, U16, 2),   # cfg4
        ((2, 7680, 4320, 1920, 1080, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),    (DIL56,) * 2, (DIL56,) * 2, SRGB, 0),   # cfg5
        ((1, 7680, 4320, 3840, 2160, 4, u8, u8, 8, {}),                             (INL24,) * 2, (INL24,) * 2, U8,  2),
        ((2, 7680, 4320, 3840, 2160, 4, f32, u16, 16, {"gamma": True}),             (0, DIL24),  (0, DIL24),   SRGB, 0),   # float + gamma source: tile row pass
        ((1, 1500, 1000, 1111, 741, 4, u8, u8, 8, {}),                              (0, 0),      (0, 0),       U8,   2),   # irregular ratio
    ]
    for case, want_def, want_all, src, epi in table:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        rs, v = cs.resizer_and_vars(case)
        h, dp, modes = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, v)
        try:
            out = (C.c_int * 4)()
            emul.stream_emul_selection(dp, 0, out)
            assert (out[0], out[1]) == want_def, (cs.case_id(case), list(out))
            if out[0]:
                assert out[2] == src, (cs.case_id(case), list(out))
            assert out[3] == epi, (cs.case_id(case), list(out))
            emul.stream_emul_selection(dp, 1, out)
            assert (out[0], out[1]) == want_all, (cs.case_id(case), list(out))
        finally:
            rs.free_descriptor(h)


def test_stream_kernel_emulation_fuzz(emul):
    """Seeded random sweep over the streaming-eligible call shapes (k = 2, 4, 2x4, 0.5; the three
    classes; both build modes; u8 / u16 / float sources and destinations; input / output gamma
    and the alpha exemption) with random warp counts, destination bands and scheduling
    variants: emulation == port on every call the streaming kernel accepts."""
    lut = np.zeros(256, np.float32)
    cs.port().avir_port_srgb_lut(lut.ctypes.data)
    rng = np.random.default_rng(5)
    types = [u8, u16, f32]
    ran = 0
    for it in range(110):
        fp, fam = int(rng.integers(0, 3)), int(rng.integers(0, 4))
        nw, nh = int(rng.integers(3, 90)), int(rng.integers(3, 60))
        if fam == 0:
            sw, sh, bm = nw * 2, nh * 2, int(rng.integers(0, 2))
        elif fam == 1:
            sw, sh, bm = nw * 4, nh * 4, int(rng.integers(0, 2))
        elif fam == 2:
            sw, sh, bm = nw * 2, nh * 4, int(rng.integers(0, 2))
        else:
            sw, sh, nw, nh, bm = nw, nh, nw * 2, nh * 2, 1
        ti, to = types[int(rng.integers(0, 3))], types[int(rng.integers(0, 3))]
        rb = int(rng.integers(5, 9)) if to == u8 else (int(rng.integers(9, 17)) if to == u16 else int(rng.choice([8, 16])))
        kw = {"buildmode": bm}
        if rng.random() < 0.4:
            kw["gamma"] = True
        if rng.random() < 0.5:
            kw["alpha"] = int(rng.choice([0, 3]))
        case = (fp, sw, sh, nw, nh, 4, ti, to, rb, kw)
        src = cs.make_input(case, seed=77 + it)
        rs, v = cs.resizer_and_vars(case)
        h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, 0.0, v)
        try:
            if emul.stream_emul_applicable(dp) != 1:
                continue
            got = np.zeros((nh, nw, 4), to)
            wh, wv = int(rng.integers(1, 9)), int(rng.integers(1, 9))
            bands, var = int(rng.integers(1, 5)), int(rng.integers(0, 4))
            assert emul.stream_emul_resize(dp, src.ctypes.data, sw * 4, got.ctypes.data, nw * 4, wh, wv, bands,
                                           var, lut.ctypes.data, 1 + (it & 1), band_needs(dp, bands), int(rng.integers(0, 20)), int(rng.integers(0, 20))) == 0
        finally:
            rs.free_descriptor(h)
        want, _ = cs.port_output(case, src)
        assert cs.count_mismatch(want, got) == 0, (cs.case_id(case), wh, wv, bands, var)
        ran += 1
    assert ran >= 30


# The value domain (cases.value_image): samples outside [0, 1], beyond int32 once scaled to the
# output range, non-finite and subnormal, through the output stage of every chain.  The emulation's
# float-to-int conversions model the device's (NaN to 0, saturating), so this is where a difference
# from upstream's x86 conversions shows up without a GPU.
VALUE_EMUL_CASES = [
    ((0, 100, 70, 50, 35, 4, f32, u8, 8, {"buildmode": 1}), 4, 3, 2),      # default class, k = 2
    ((0, 256, 192, 128, 96, 4, f32, u8, 8, {"buildmode": 1}), 3, 2, 1),    # every huge patch
    ((0, 256, 192, 128, 96, 4, f32, u16, 16, {"buildmode": 1}), 2, 5, 3),
    ((0, 128, 96, 256, 192, 4, f32, u16, 16, {"buildmode": 1}), 3, 2, 1),  # cfg2 chain
    ((0, 256, 192, 64, 48, 4, f32, u8, 8, {"buildmode": 0}), 2, 2, 2),     # cfg4 chain
    ((1, 256, 192, 128, 96, 4, f32, u8, 8, {"buildmode": 1}), 4, 3, 2),    # RNE_I32
    ((1, 256, 192, 64, 48, 4, f32, u16, 16, {"buildmode": 0}), 3, 2, 1),
    ((2, 256, 192, 128, 96, 4, f32, u16, 16, {"buildmode": 1}), 2, 2, 1),  # RNE
    ((2, 256, 192, 64, 48, 4, f32, u8, 8, {"buildmode": 1}), 3, 4, 2),     # cfg5 chain
    ((2, 256, 192, 128, 96, 4, f32, f32, 16, {"buildmode": 1}), 3, 2, 1),  # float output
    ((1, 256, 192, 128, 96, 4, f32, f32, 16, {"buildmode": 0}), 2, 3, 2),
]


@pytest.mark.parametrize("kind", ("range", "huge", "nonfinite", "tiny"))
@pytest.mark.parametrize("ec", VALUE_EMUL_CASES, ids=_id)
def test_stream_kernel_emulation_value_domain(emul, ec, kind):
    case, wh, wv, bands = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.value_image(case, kind)
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        assert emul.stream_emul_applicable(dp) == 1, "chain not on the streaming kernel: %r" % (modes,)
        got = np.zeros((nh, nw, ch), to)
        lut = np.zeros(256, np.float32)
        cs.port().avir_port_srgb_lut(lut.ctypes.data)
        assert emul.stream_emul_resize(dp, src.ctypes.data, sw * ch, got.ctypes.data, nw * ch, wh, wv, bands,
                                       1, lut.ctypes.data, 1, band_needs(dp, bands), wh % 7, wv % 5) == 0
    finally:
        rs.free_descriptor(h)
    want, _ = cs.port_output(case, src)
    assert cs.value_mismatch(want, got) == 0


# Caller layouts: the source rows padded (pitch % 4 == 0 keeps the pass on the streaming kernel) with
# poison in the padding, the destination rows padded and every byte outside the image a sentinel.
@pytest.mark.parametrize("fused", [False, True], ids=["copied-halo", "fused"])
@pytest.mark.parametrize("ec", EMUL_CASES[::5], ids=_id)
def test_stream_kernel_emulation_padded_pitches(emul, ec, fused):
    case, wh, wv, bands = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    if fused:
        bands = max(bands, 2)
    src = cs.make_input(case)
    sl = cs.source_layout(src, 12)
    dl = cs.guarded_dest((nh, nw, ch), to, 10)
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        lut = np.zeros(256, np.float32)
        cs.port().avir_port_srgb_lut(lut.ctypes.data)
        s_ptr, d_ptr = sl.view().ctypes.data, dl.view().ctypes.data
        if fused:
            infos = band_infos(dp, bands)
            if infos is None:
                pytest.skip("bands too small for the sharded schedule")
            rc = emul.stream_emul_resize_fused(dp, s_ptr, sl.pitch, d_ptr, dl.pitch, wh, wv, bands, 0,
                                               lut.ctypes.data, 1, infos)
            if rc == 1:
                pytest.skip("a strip with rows of both neighbours: the product pushes with the copy engines")
            assert rc == 0
        else:
            assert emul.stream_emul_resize(dp, s_ptr, sl.pitch, d_ptr, dl.pitch, wh, wv, bands, 1,
                                           lut.ctypes.data, 1, band_needs(dp, bands), wh % 7, wv % 5) == 0
    finally:
        rs.free_descriptor(h)
    want, _ = cs.port_output(case, src)
    assert cs.count_mismatch(want, np.ascontiguousarray(dl.view())) == 0
    assert cs.guard_damage(dl) == 0
