"""Destination windows without a GPU: the footprint avirb200_window_query_desc reports, and the windowed
streaming passes in the host emulation.

A window (x0, y0, w, h) of a plan's full resize must equal the same pixels of the whole image.  The
footprint is checked on the oracle's C port: a source that is poisoned everywhere outside the footprint
must give the window the same bits as the clean source.  The streaming kernel's windowed row pass (the
output column range, a source buffer whose column 0 is the footprint's) is checked in the lockstep
emulation (tests/emul/window_emul.cpp) on buffers exactly the footprint's and the window's size, with
every read bounds-checked, against the port's whole image."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs

u8, u16, f32 = np.uint8, np.uint16, np.float32
ERR_BAD_ARG, ERR_UNSUPPORTED = -1, -4


class WindowInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_x0", "src_w", "src_y0", "src_h", "mid_row0", "mid_rows")]


def window_query_desc(dp, win):
    info = WindowInfo()
    rc = ab.lib().avirb200_window_query_desc(C.c_void_p(dp), *[int(v) for v in win], C.byref(info))
    return rc, info


def window_set(nw, nh, seed=3):
    """1x1 at each corner and the centre, single rows and columns, windows on each image edge, left edges
    inside the first and the last round of a streaming run (the round lengths are 4..32 outputs), and a
    seeded random set."""
    rng = np.random.default_rng(seed)
    ws = [(0, 0, 1, 1), (nw - 1, 0, 1, 1), (0, nh - 1, 1, 1), (nw - 1, nh - 1, 1, 1), (nw // 2, nh // 2, 1, 1),
          (0, nh // 3, nw, 1), (nw // 4, nh - 1, max(1, nw // 2), 1),
          (nw // 3, 0, 1, nh), (nw - 1, nh // 4, 1, max(1, nh // 2)),
          (0, 0, nw, nh)]
    for _ in range(2):
        w, h = int(rng.integers(1, nw + 1)), int(rng.integers(1, nh + 1))
        x, y = int(rng.integers(0, nw - w + 1)), int(rng.integers(0, nh - h + 1))
        ws += [(0, y, w, h), (nw - w, y, w, h), (x, 0, w, h), (x, nh - h, w, h)]
    for x0 in (1, 3, 5, 9, 17, 31):   # inside a run's first round ...
        if x0 < nw:
            w = int(rng.integers(1, nw - x0 + 1))
            ws.append((x0, int(rng.integers(0, nh)), w, 1 + int(rng.integers(0, nh)) // 2))
    for back in (2, 6, 13):           # ... and its last (left and right edges)
        if back < nw:
            x1 = nw - back
            x0 = int(rng.integers(0, x1))
            ws += [(nw - back, nh // 5, back, 2), (x0, nh // 2, x1 - x0, 1 + nh // 7)]
    for _ in range(6):
        w, h = int(rng.integers(1, nw + 1)), int(rng.integers(1, nh + 1))
        ws.append((int(rng.integers(0, nw - w + 1)), int(rng.integers(0, nh - h + 1)), w, h))
    out = []
    for (x, y, w, h) in ws:
        x, y = max(0, min(x, nw - 1)), max(0, min(y, nh - 1))
        w, h = max(1, min(w, nw - x)), max(1, min(h, nh - y))
        if (x, y, w, h) not in out:
            out.append((x, y, w, h))
    return out


def crop(img, win):
    x, y, w, h = win
    return np.ascontiguousarray(img[y:y + h, x:x + w])


def _poisons(dtype):
    dtype = np.dtype(dtype)
    return (np.nan,) if dtype.kind == "f" else (0, np.iinfo(dtype).max)


def _is_errd(case):
    return case[0] >= 3 and np.dtype(case[7]).kind != "f"


@pytest.mark.parametrize("case", [c for c in cs.SMALL_CASES if not _is_errd(c)], ids=cs.case_id)
def test_window_footprint_holds_every_source_pixel_the_window_reads(case):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        full = np.zeros((nh, nw, ch), to)
        assert cs.port().avir_port_resize(dp, src.ctypes.data, sw * ch, full.ctypes.data, nw * ch) == 0
        for win in window_set(nw, nh):
            rc, fi = window_query_desc(dp, win)
            assert rc == 0, (win, ab.lib().avirb200_last_error())
            assert 0 <= fi.src_x0 and fi.src_w >= 1 and fi.src_x0 + fi.src_w <= sw, win
            assert 0 <= fi.src_y0 and fi.src_h >= 1 and fi.src_y0 + fi.src_h <= sh, win
            assert (fi.mid_row0, fi.mid_rows) == (fi.src_y0, fi.src_h)
            for poison in _poisons(ti):
                bad = np.full_like(src, poison)
                ys, xs = slice(fi.src_y0, fi.src_y0 + fi.src_h), slice(fi.src_x0, fi.src_x0 + fi.src_w)
                bad[ys, xs] = src[ys, xs]
                got = np.zeros((nh, nw, ch), to)
                assert cs.port().avir_port_resize(dp, bad.ctypes.data, sw * ch, got.ctypes.data, nw * ch) == 0
                assert cs.count_mismatch(crop(full, win), crop(got, win)) == 0, (win, poison)
    finally:
        rs.free_descriptor(h)


def test_window_footprint_of_a_full_size_chain():
    """cfg4's geometry (16384^2 -> 4096^2): a 1920x1080 window reads about an eighth of the source."""
    case = (1, 16384, 16384, 4096, 4096, 4, u16, u16, 16, {})
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((16384, 16384, 4), u16, 4096, 4096, u16, 0.0, v)
    try:
        rc, fi = window_query_desc(dp, (1001, 1503, 1920, 1080))
        assert rc == 0
        # the window's own source pixels (4x) plus the chain's reach on either side
        assert 4 * 1920 < fi.src_w < 4 * 1920 + 128 and 4 * 1080 < fi.src_h < 4 * 1080 + 128
        assert abs(fi.src_x0 - 4 * 1001) < 64 and abs(fi.src_y0 - 4 * 1503) < 64
        rc, fi = window_query_desc(dp, (0, 0, 4096, 4096))
        assert (rc, fi.src_x0, fi.src_w, fi.src_y0, fi.src_h) == (0, 0, 16384, 0, 16384)
    finally:
        rs.free_descriptor(h)


def test_window_query_desc_rejects_bad_windows():
    case = (2, 192, 108, 96, 54, 4, f32, f32, 16, {})
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((108, 192, 4), f32, 96, 54, f32, 0.0, v)
    try:
        for win in [(0, 0, 0, 1), (0, 0, 1, 0), (-1, 0, 4, 4), (0, -1, 4, 4), (93, 0, 4, 4), (0, 51, 4, 4),
                    (96, 0, 1, 1), (0, 54, 1, 1), (2 ** 31 - 1, 0, 2, 1), (0, 2 ** 31 - 1, 1, 2),
                    (1, 1, 2 ** 31 - 1, 1), (0, 0, -5, 3)]:
            assert window_query_desc(dp, win)[0] == ERR_BAD_ARG, win
        assert window_query_desc(dp, (0, 0, 96, 54))[0] == 0
        assert ab.lib().avirb200_window_query_desc(None, 0, 0, 1, 1, None) == ERR_BAD_ARG
    finally:
        rs.free_descriptor(h)


@pytest.mark.parametrize("fp", (3, 4, 5))
def test_window_query_desc_refuses_error_diffusion(fp):
    case = (fp, 120, 80, 60, 40, 4, u8, u8, 8, {})
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((80, 120, 4), u8, 60, 40, u8, 0.0, v)
    try:
        assert window_query_desc(dp, (3, 4, 10, 10))[0] == ERR_UNSUPPORTED
        assert window_query_desc(dp, (3, 4, 0, 10))[0] == ERR_BAD_ARG   # a bad window first
    finally:
        rs.free_descriptor(h)
    # float output skips the ditherer: windows are fine
    rs, v = cs.resizer_and_vars((fp, 120, 80, 60, 40, 4, u8, f32, 8, {}))
    h, dp, _ = rs.descriptor((80, 120, 4), u8, 60, 40, f32, 0.0, v)
    try:
        assert window_query_desc(dp, (3, 4, 10, 10))[0] == 0
    finally:
        rs.free_descriptor(h)


# ---- the windowed streaming passes in the host emulation -------------------------------------------------

@pytest.fixture(scope="module")
def wemul():
    from avir_b200 import build as b
    lib = C.CDLL(b.build_window_emul())
    lib.stream_emul_window.argtypes = ([C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t] + [C.c_int] * 4 +
                                       [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p, C.c_int, C.c_int])
    lib.stream_emul_window.restype = C.c_int
    return lib


# (case, emulated warps of the row pass, of the column pass): every streaming chain and source type
EMUL_WINDOW_CASES = [
    ((2, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1}), 3, 2),     # cfg3 chain (DIL mirror)
    ((1, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 0}), 4, 3),     # cfg3 chain (float4 mirror)
    ((1, 100, 70, 50, 35, 4, f32, u8, 8, {"buildmode": 1}), 2, 5),        # k = 2, mode 1; integer output
    ((1, 96, 54, 192, 108, 4, u8, u8, 8, {"buildmode": 1}), 3, 2),        # cfg2 chain, u8 source
    ((1, 384, 216, 96, 54, 4, u16, u16, 16, {"buildmode": 0}), 3, 2),     # cfg4 chain
    ((2, 384, 216, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3, "buildmode": 1}), 5, 3),  # cfg5, sRGB source
]


def _eid(ec):
    return "%s-w%d-%d" % (cs.case_id(ec[0]), ec[1], ec[2])


def _emul_window(wemul, dp, src, to, win, fi, wh, wv, variant, ignore_cols=0):
    ch = src.shape[2]
    fsrc = np.ascontiguousarray(src[fi.src_y0:fi.src_y0 + fi.src_h, fi.src_x0:fi.src_x0 + fi.src_w])
    got = np.zeros((win[3], win[2], ch), to)
    lut = np.zeros(256, np.float32)
    cs.port().avir_port_srgb_lut(lut.ctypes.data)
    fp = (C.c_int * 4)(fi.src_x0, fi.src_w, fi.src_y0, fi.src_h)
    rc = wemul.stream_emul_window(dp, fsrc.ctypes.data, fi.src_w * ch, got.ctypes.data, win[2] * ch, *win, fp, wh, wv,
                                  variant, lut.ctypes.data, 1, ignore_cols)
    return rc, got


@pytest.mark.parametrize("variant", range(4))
@pytest.mark.parametrize("ec", EMUL_WINDOW_CASES, ids=_eid)
def test_stream_window_emulation_matches_port(wemul, ec, variant):
    case, wh, wv = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    want, _ = cs.port_output(case, src)
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor(src.shape, src.dtype, nw, nh, to, 0.0, v)
    try:
        for win in window_set(nw, nh, seed=variant):
            rc, fi = window_query_desc(dp, win)
            assert rc == 0
            rc, got = _emul_window(wemul, dp, src, to, win, fi, wh, wv, variant)
            assert rc == 0, (win, rc)
            assert cs.count_mismatch(crop(want, win), got) == 0, win
    finally:
        rs.free_descriptor(h)


@pytest.mark.parametrize("ec", EMUL_WINDOW_CASES[:3], ids=_eid)
def test_stream_window_emulation_catches_a_row_pass_without_the_column_range(wemul, ec):
    """The same check against a row pass that reads the footprint buffer as if it held the whole line:
    every window away from the left edge must fail (a read outside the buffer, or wrong bits)."""
    case, wh, wv = ec
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    want, _ = cs.port_output(case, src)
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor(src.shape, src.dtype, nw, nh, to, 0.0, v)
    try:
        caught = 0
        wins = [w for w in window_set(nw, nh) if window_query_desc(dp, w)[1].src_x0 > 0]
        assert len(wins) >= 8
        for win in wins:
            fi = window_query_desc(dp, win)[1]
            rc, got = _emul_window(wemul, dp, src, to, win, fi, wh, wv, 1, ignore_cols=1)
            caught += (rc == -5 or cs.count_mismatch(crop(want, win), got) > 0)
        assert caught == len(wins)
    finally:
        rs.free_descriptor(h)
