"""CLancIR destination windows without a GPU: the footprint lancirb200_window_query_desc reports.

A window (x0, y0, w, h) of a LANCIR resize must equal the same pixels of the whole image, reading only its
footprint: per axis, the min / max of every tap position of the window's outputs clamped to the image.
The footprint is checked against that rule computed by brute force, and on the oracle's C port
(lancir_port_resize): a source poisoned everywhere outside the footprint must give the window the same
bits as the clean source.  NaN poison catches zero-valued taps too (the kernels multiply every tap, and
0 * NaN is NaN), so it also shows that their positions lie inside the footprint."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_window import crop, window_set

u8, u16, f32 = np.uint8, np.uint16, np.float32
ERR_BAD_ARG = -1


class LancirAxis(C.Structure):
    _fields_ = [("src_len", C.c_int32), ("dst_len", C.c_int32), ("kernel_len", C.c_int32), ("nphases", C.c_int32),
                ("taps", C.POINTER(C.c_float)), ("src_pos", C.POINTER(C.c_int32)), ("phase", C.POINTER(C.c_int32))]


class LancirDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_w", "src_h", "dst_w", "dst_h", "channels", "in_type", "out_type")] + [
        ("out_mul", C.c_float), ("is_unity_mul", C.c_int32), ("clamp_max", C.c_float),
        ("v", LancirAxis), ("h", LancirAxis)]


class LancirWindowInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_x0", "src_w", "src_y0", "src_h")]


# (sw, sh, nw, nh, channels, Tin, Tout, CLancIRParams fields): 1-4 channels, la 2-5, upsizing (6 taps),
# k = 2 / 3 / 4, explicit and negative k, offsets
CASES = [
    (96, 54, 48, 27, 4, u8, u8, {}),                                        # k = 2: 12 taps
    (64, 48, 103, 77, 4, u8, u8, {}),                                       # upsizing: 6 taps
    (60, 45, 20, 15, 3, u8, u8, {}),                                        # k = 3: 18 taps
    (64, 64, 16, 16, 4, u16, u16, {}),                                      # k = 4: 24 taps
    (50, 30, 33, 17, 4, f32, u8, {}),
    (77, 51, 47, 29, 3, f32, f32, {"kx": 1.3, "ky": 2.2}),
    (96, 54, 48, 27, 1, u8, f32, {}),
    (77, 51, 50, 31, 2, u16, u16, {"la": 2.0}),
    (77, 51, 47, 29, 1, f32, u16, {"la": 5.0, "kx": -1.3, "ky": -0.9, "ox": 0.25, "oy": -0.5}),
    (50, 30, 70, 45, 2, u8, f32, {"kx": 0.7, "ky": -0.66, "ox": 0.25, "oy": 0.1}),
    (33, 21, 7, 5, 3, u8, u8, {"la": 4.0}),
    (40, 30, 40, 30, 4, f32, f32, {"ox": 3.5, "oy": -2.25}),               # taps pushed off the image
]


def case_id(c):
    sw, sh, nw, nh, ch, ti, to, kw = c
    s = "%dx%d-%dx%d-c%d-%s-%s" % (sw, sh, nw, nh, ch, np.dtype(ti).name, np.dtype(to).name)
    return s + "".join("-%s%s" % kv for kv in sorted(kw.items()))


class Descriptor:
    """The descriptor CLancIR::resizeImage builds for the case (host only)."""

    def __init__(self, c):
        sw, sh, nw, nh, ch, ti, to, kw = c
        self.handle = ab.host_lib().lancirb200_host_desc_create(
            o.T_OF[np.dtype(ti)], o.T_OF[np.dtype(to)], sw, sh, nw, nh, ch, kw.get("kx", 0.0), kw.get("ky", 0.0),
            kw.get("ox", 0.0), kw.get("oy", 0.0), kw.get("la", 3.0))
        assert self.handle
        self.ptr = ab.host_lib().lancirb200_host_desc_get(self.handle)
        self.desc = LancirDesc.from_address(self.ptr)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        ab.host_lib().lancirb200_host_desc_free(self.handle)


def query_desc(dp, win):
    info = LancirWindowInfo()
    rc = ab.lib().lancirb200_window_query_desc(C.c_void_p(dp), *[int(v) for v in win], C.byref(info))
    return rc, info


def brute_span(ax, i0, n):
    """[lo, hi] of every tap position of outputs i0 .. i0 + n - 1, clamped to [0, src_len)."""
    pos = np.ctypeslib.as_array(ax.src_pos, (ax.dst_len,)).astype(np.int64)[i0:i0 + n]
    taps = np.clip(pos[:, None] + np.arange(ax.kernel_len)[None, :], 0, ax.src_len - 1)
    return int(taps.min()), int(taps.max())


def check_brute_force(d, dp, win):
    rc, fi = query_desc(dp, win)
    assert rc == 0, (win, ab.lib().avirb200_last_error())
    x0, y0, w, h = win
    assert (fi.src_x0, fi.src_x0 + fi.src_w - 1) == brute_span(d.h, x0, w), win
    assert (fi.src_y0, fi.src_y0 + fi.src_h - 1) == brute_span(d.v, y0, h), win
    return fi


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_footprint_is_the_span_of_the_clamped_taps(c):
    sw, sh, nw, nh, ch, ti, to, kw = c
    with Descriptor(c) as dd:
        for win in window_set(nw, nh):
            check_brute_force(dd.desc, dd.ptr, win)


def _poisons(dtype):
    dtype = np.dtype(dtype)
    return (np.nan,) if dtype.kind == "f" else (0, np.iinfo(dtype).max)


def port_resize(dp, src, nw, nh, to):
    sh, sw, ch = src.shape
    out = np.zeros((nh, nw, ch), to)
    assert cs.port().lancir_port_resize(dp, src.ctypes.data, sw * ch, out.ctypes.data, nw * ch) == 0
    return out


def check_poisoned(dp, src, nw, nh, to, wins):
    full = port_resize(dp, src, nw, nh, to)
    for win in wins:
        rc, fi = query_desc(dp, win)
        assert rc == 0
        for poison in _poisons(src.dtype):
            bad = np.full_like(src, poison)
            ys, xs = slice(fi.src_y0, fi.src_y0 + fi.src_h), slice(fi.src_x0, fi.src_x0 + fi.src_w)
            bad[ys, xs] = src[ys, xs]
            got = port_resize(dp, bad, nw, nh, to)
            assert cs.count_mismatch(crop(full, win), crop(got, win)) == 0, (win, poison)


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_footprint_holds_every_source_pixel_the_window_reads(c):
    sw, sh, nw, nh, ch, ti, to, kw = c
    src = o.lcg_image(sh, sw, ch, ti, seed=21)
    with Descriptor(c) as dd:
        check_poisoned(dd.ptr, src, nw, nh, to, window_set(nw, nh, seed=4))


def test_footprint_does_not_assume_monotone_tables():
    """A descriptor whose positions jump back and forth (the C ABI accepts any table): the footprint is
    the min / max over the window's entries, not its first and last output's."""
    c = (60, 40, 30, 20, 3, f32, f32, {})
    sw, sh, nw, nh, ch, ti, to, kw = c
    rng = np.random.default_rng(5)
    with Descriptor(c) as dd:
        d = dd.desc
        for ax in (d.h, d.v):
            pos = np.ctypeslib.as_array(ax.src_pos, (ax.dst_len,))
            pos[:] = rng.permutation(pos)
            pos[ax.dst_len // 2] = -3 * ax.kernel_len        # wholly before the image
            pos[ax.dst_len // 3] = ax.src_len + 7             # wholly after it
        wins = window_set(nw, nh, seed=8)
        for win in wins:
            check_brute_force(d, dd.ptr, win)
        check_poisoned(dd.ptr, o.lcg_image(sh, sw, ch, ti, seed=22), nw, nh, to, wins[::2])


def test_footprint_of_a_full_size_window():
    """8K -> 4K RGBA: a 1920 x 1080 window at odd offsets reads its own source pixels (2x) plus the
    12-tap kernel's reach, about a quarter of the source."""
    c = (7680, 4320, 3840, 2160, 4, u8, u8, {})
    with Descriptor(c) as dd:
        win = ((3840 - 1920) // 2 + 1, (2160 - 1080) // 2 + 1, 1920, 1080)
        fi = check_brute_force(dd.desc, dd.ptr, win)
        assert (fi.src_w, fi.src_h) == (2 * 1920 + 10, 2 * 1080 + 10)
        assert (fi.src_x0, fi.src_y0) == (2 * win[0] - 5, 2 * win[1] - 5)
        rc, fi = query_desc(dd.ptr, (0, 0, 3840, 2160))
        assert (rc, fi.src_x0, fi.src_w, fi.src_y0, fi.src_h) == (0, 0, 7680, 0, 4320)


BAD_WINDOWS = [(0, 0, 0, 1), (0, 0, 1, 0), (-1, 0, 4, 4), (0, -1, 4, 4), (45, 0, 4, 4), (0, 24, 4, 4),
               (48, 0, 1, 1), (0, 27, 1, 1), (2 ** 31 - 1, 0, 2, 1), (0, 2 ** 31 - 1, 1, 2),
               (1, 1, 2 ** 31 - 1, 1), (0, 0, -5, 3), (0, 0, 49, 1), (0, 0, 1, 28)]


def test_bad_windows_are_refused_without_a_device():
    with Descriptor((96, 54, 48, 27, 4, u8, u8, {})) as dd:
        for win in BAD_WINDOWS:
            assert query_desc(dd.ptr, win)[0] == ERR_BAD_ARG, win
        assert query_desc(dd.ptr, (0, 0, 48, 27))[0] == 0
        assert query_desc(dd.ptr, (47, 26, 1, 1))[0] == 0
    L = ab.lib()
    info = LancirWindowInfo()
    assert L.lancirb200_window_query_desc(None, 0, 0, 1, 1, C.byref(info)) == ERR_BAD_ARG
    vp, i = C.c_void_p, C.c_int
    L.lancirb200_window_query.argtypes = [vp, i, i, i, i, vp]
    L.lancirb200_window_workspace_bytes.argtypes = [vp, i, i, i, i, vp]
    L.lancirb200_resize_window_device.argtypes = [vp, i, i, i, i, vp, C.c_size_t, vp, C.c_size_t, vp, vp]
    L.lancirb200_resize_window_host.argtypes = [vp, i, i, i, i, vp, C.c_size_t, vp, C.c_size_t]
    assert L.lancirb200_window_query(None, 0, 0, 1, 1, C.byref(info)) == ERR_BAD_ARG
    n = C.c_size_t()
    assert L.lancirb200_window_workspace_bytes(None, 0, 0, 1, 1, C.byref(n)) == ERR_BAD_ARG
    buf = np.zeros(64, u8)
    assert L.lancirb200_resize_window_device(None, 0, 0, 1, 1, buf.ctypes.data, 4, buf.ctypes.data, 4,
                                             buf.ctypes.data, None) == ERR_BAD_ARG
    assert L.lancirb200_resize_window_host(None, 0, 0, 1, 1, buf.ctypes.data, 4, buf.ctypes.data, 4) == ERR_BAD_ARG


def test_front_end_refuses_bad_windows_without_a_device():
    """CLancIR::resizeImageWindow keeps upstream's error convention: 0 for bad arguments, before any CUDA
    call."""
    src = o.lcg_image(54, 96, 4, u8, seed=1)
    lr = ab.CLancIR()
    for win in BAD_WINDOWS:
        if win[2] > 0 and win[3] > 0 and win[2] * win[3] < 4096:
            r, _ = lr.resizeImageWindow(src, 48, 27, *win)
            assert r == 0, win
    assert lr.resizeImageWindow(src, 48, 27, 0, 0, 4, 4, ab.CLancIRParams(la=1.5))[0] == 0
    assert lr.windowFootprint(src.shape, u8, 48, 27, u8, (45, 0, 4, 4)) is None
    assert lr.windowWorkspaceBytes(src.shape, u8, 48, 27, u8, (0, 0, 0, 4)) == 0


def test_front_end_zero_fills_the_window_of_an_empty_source():
    """lancir.h:414-426 for the window's pixels: a 0-sized source gives a zero window (no device needed);
    NewSSize padding is left alone."""
    lr = ab.CLancIR()
    back = np.full((5, 12, 3), 7, u8)
    view = back[:, :10, :]   # rows 36 elements apart, the window 10 pixels wide
    r, _ = lr.resizeImageWindow(np.zeros((0, 0, 3), u8), 40, 30, 3, 4, 10, 5, ab.CLancIRParams(NewSSize=36),
                                NewBuf=view)
    assert r == 5
    assert (back[:, :10] == 0).all() and (back[:, 10:] == 7).all()
