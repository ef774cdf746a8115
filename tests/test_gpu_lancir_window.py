"""CLancIR destination windows on the GPU (run with -m gpu on an H100): lancirb200_resize_window_device /
_host and CLancIR::resizeImageWindow* against the whole image.

A window (x0, y0, w, h) must equal the same pixels of lancirb200_resize_device on the whole image (and
upstream's output where oracle/_ref is present), with the source buffer holding the window's footprint.
Buffer layouts follow test_gpu_layouts.py: poisoned source guards, sentinel destination guards and a
sentinel tail behind the workspace the library asked for."""
import contextlib
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_gpu_layouts import LANCIR_CASES as LAYOUT_CASES
from test_gpu_layouts import LANCIR_LAYOUTS, _ok, _src_pitch, guarded_workspace, launched_kernels, tail_damage
from test_gpu_parity import LANCIR as PARITY_CASES
from test_gpu_window import footprint_layout, upload
from test_lancir_window import LancirWindowInfo
from test_window import crop, window_set

pytestmark = pytest.mark.gpu

u8, u16, f32 = np.uint8, np.uint16, np.float32
TYPES = (u8, u16, f32)
ERR_BAD_ARG, ERR_UNSUPPORTED = -1, -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def llib():
    L = ab.lib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    L.lancirb200_plan_workspace_bytes.argtypes = [vp, vp]
    L.lancirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    L.lancirb200_window_query.argtypes = [vp, i, i, i, i, vp]
    L.lancirb200_window_workspace_bytes.argtypes = [vp, i, i, i, i, vp]
    L.lancirb200_resize_window_device.argtypes = [vp, i, i, i, i, vp, sz, vp, sz, vp, vp]
    L.lancirb200_resize_window_host.argtypes = [vp, i, i, i, i, vp, sz, vp, sz]
    return L


@contextlib.contextmanager
def lancir_plan(sw, sh, nw, nh, ch, ti, to, kw):
    """A C-ABI plan of the call, as CLancIR::resizeImage builds it; yields (library, plan, descriptor)."""
    h = ab.host_lib().lancirb200_host_desc_create(o.T_OF[np.dtype(ti)], o.T_OF[np.dtype(to)], sw, sh, nw, nh, ch,
                                                  kw.get("kx", 0.0), kw.get("ky", 0.0), kw.get("ox", 0.0),
                                                  kw.get("oy", 0.0), kw.get("la", 3.0))
    assert h
    L, pl = llib(), C.c_void_p()
    dp = ab.host_lib().lancirb200_host_desc_get(h)
    try:
        _ok(L.lancirb200_plan_create(C.c_void_p(dp), C.byref(pl)))
        yield L, pl, dp
    finally:
        if pl.value:
            L.lancirb200_plan_destroy(pl)
        ab.host_lib().lancirb200_host_desc_free(h)


def query(L, pl, win):
    fi, n = LancirWindowInfo(), C.c_size_t()
    _ok(L.lancirb200_window_query(pl, *win, C.byref(fi)))
    _ok(L.lancirb200_window_workspace_bytes(pl, *win, C.byref(n)))
    return fi, n.value


def full_device(L, pl, d_src, sw, sh, nw, nh, ch, to):
    """lancirb200_resize_device on the whole image (packed buffers)."""
    import torch
    n = C.c_size_t()
    _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
    d_dst = torch.empty(nh * nw * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
    ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
    _ok(L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch, ws.data_ptr(), None))
    torch.cuda.synchronize()
    return d_dst.cpu().numpy().view(to).reshape(nh, nw, ch)


def window_in_place(L, pl, d_src, sw, ch, ti, to, win):
    """The window with d_src pointing at its footprint inside the whole device image (pitched)."""
    import torch
    fi, n = query(L, pl, win)
    d_dst = torch.empty(win[2] * win[3] * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
    ws = torch.empty(n, dtype=torch.uint8, device="cuda")
    src_ptr = d_src.data_ptr() + (fi.src_y0 * sw + fi.src_x0) * ch * np.dtype(ti).itemsize
    _ok(L.lancirb200_resize_window_device(pl, *win, src_ptr, sw * ch, d_dst.data_ptr(), win[2] * ch, ws.data_ptr(),
                                          None))
    torch.cuda.synchronize()
    return d_dst.cpu().numpy().view(to).reshape(win[3], win[2], ch)


def check_windows(src, nw, nh, to, kw, wins, mismatch=cs.count_mismatch, ref=None):
    sh, sw, ch = src.shape
    with lancir_plan(sw, sh, nw, nh, ch, src.dtype, to, kw) as (L, pl, _):
        d_src = upload(src)
        full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, to)
        if ref is not None:
            assert mismatch(ref, full) == 0
        for win in wins:
            got = window_in_place(L, pl, d_src, sw, ch, src.dtype, to, win)
            assert mismatch(crop(full, win), got) == 0, win
    return full


# ---- equality with the whole image: every LANCIR case x every type pair x the window set ----------------------

def _geometries():
    out = []
    for sw, sh, nw, nh, ti, to, kw in PARITY_CASES + LAYOUT_CASES:
        kw = dict(kw)
        g = (sw, sh, nw, nh, kw.pop("C", 4), tuple(sorted(kw.items())))
        if g not in out:
            out.append(g)
    return out


def _gid(g):
    return "%dx%d-%dx%d-c%d" % g[:5] + "".join("-%s%s" % kv for kv in g[5])


@pytest.mark.parametrize("to", TYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("ti", TYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("g", _geometries(), ids=_gid)
def test_window_equals_the_whole_image(g, ti, to):
    sw, sh, nw, nh, ch, kw = g
    kw = dict(kw)
    src = o.lcg_image(sh, sw, ch, ti, seed=3)
    ref = None
    if o.have_ref():
        r, ref = o.lancir_ref(src, nw, nh, to, **kw)
        assert r == nh
    check_windows(src, nw, nh, to, kw, window_set(nw, nh, seed=sw + nh), ref=ref)


# ---- the (NewWidth * C) & 3 tail: decided by the element's place in the whole row, not in the window ---------

TAIL_CASES = [(77, 51, 47, 29, 1, u8), (77, 51, 47, 29, 2, u16), (77, 51, 47, 29, 3, u8),
              (64, 48, 103, 77, 3, u16), (50, 30, 33, 17, 2, u8), (60, 40, 21, 13, 1, u16)]


def tail_windows(nw, nh, ch):
    t0 = ((nw * ch) & ~3) // ch            # first pixel with an element in the tail
    wins = []
    for w in (1, 2, 3, 5, nw - t0 + 1, nw // 2, nw):            # ending at the right edge
        w = max(1, min(w, nw))
        wins.append((nw - w, nh // 3, w, 3))
    for x in range(t0, nw):                                    # starting inside the tail
        wins.append((x, 1, nw - x, nh - 2))
        wins.append((x, 0, 1, nh))
    for x1 in (t0, t0 - 1, t0 - 2):                             # ending just before the tail
        if x1 >= 1:
            wins += [(0, 2, x1, 5), (max(0, x1 - 3), nh // 2, min(3, x1), 1)]
    wins += [(nw - 1, y, 1, 1) for y in (0, nh // 2, nh - 1)]   # 1 pixel on the last column
    return sorted(set(wins))


def _tid(c):
    return "%dx%d-%dx%d-c%d-%s" % (c[:5] + (np.dtype(c[5]).name,))


@pytest.mark.parametrize("c", TAIL_CASES, ids=_tid)
def test_tail_windows(c):
    sw, sh, nw, nh, ch, to = c
    assert (nw * ch) & 3
    wins = tail_windows(nw, nh, ch)
    for ti in TYPES:
        src = o.lcg_image(sh, sw, ch, ti, seed=8)
        ref = o.lancir_ref(src, nw, nh, to)[1] if o.have_ref() else None
        check_windows(src, nw, nh, to, {}, wins, ref=ref)


@pytest.mark.parametrize("c", TAIL_CASES, ids=_tid)
def test_tail_windows_on_ties(c):
    """A constant source on an output tie (k + 1/2 with k even, within a few ulps after the tap sums):
    nearest-even and (int)(v + 0.5f) disagree on many elements, so a window that placed the tail by its
    own width would differ from the whole image."""
    sw, sh, nw, nh, ch, to = c
    mul = 255.0 if to == u8 else 65535.0
    src = np.empty((sh, sw, ch), f32)
    for k in range(ch):
        src[..., k] = np.float32((2 * (40 + 2 * k) + 1) / (2 * mul))
    full = check_windows(src, nw, nh, to, {}, tail_windows(nw, nh, ch))
    with lancir_plan(sw, sh, nw, nh, ch, f32, f32, {}) as (L, pl, _):
        pre = full_device(L, pl, upload(src), sw, sh, nw, nh, ch, f32).reshape(nh, nw * ch) * np.float32(mul)
    rne = np.rint(pre).astype(np.int64)
    assert (full.reshape(nh, nw * ch) != rne).any(), "no element where the tail rounding matters"
    assert (full.reshape(nh, nw * ch)[:, :(nw * ch) & ~3] == rne[:, :(nw * ch) & ~3]).all()


# ---- buffer layouts: the four LANCIR_LAYOUTS on the footprint and the window; guards; routing --------------

def _layouts(src, fi, win, to, layout):
    sk, so, dmod, do = LANCIR_LAYOUTS[layout]
    ch = src.shape[2]
    sl = footprint_layout(src, fi, _src_pitch(fi.src_w * ch, sk) - fi.src_w * ch, so)
    p = win[2] * ch + 4
    p += (dmod - p) % 4
    return sl, cs.guarded_dest((win[3], win[2], ch), to, p - win[2] * ch, do)


def run_layout(L, pl, src, fi, n, win, to, layout):
    import torch
    sl, dl = _layouts(src, fi, win, to, layout)
    d_src, d_dst, ws = upload(sl.backing), upload(dl.backing), guarded_workspace(n)
    es, eo = src.dtype.itemsize, np.dtype(to).itemsize

    def call():
        _ok(L.lancirb200_resize_window_device(pl, *win, d_src.data_ptr() + sl.origin * es, sl.pitch,
                                              d_dst.data_ptr() + dl.origin * eo, dl.pitch, ws.data_ptr(), None))
    call()
    torch.cuda.synchronize()
    return sl, dl, d_src, d_dst, ws, call


@pytest.mark.parametrize("layout", list(LANCIR_LAYOUTS))
@pytest.mark.parametrize("c", LAYOUT_CASES, ids=lambda c: "%dx%d-%dx%d-%s-%s-c%d" % (
    c[:4] + (np.dtype(c[4]).name, np.dtype(c[5]).name, c[6].get("C", 4))))
def test_window_buffer_layouts(c, layout):
    sw, sh, nw, nh, ti, to, kw = c
    kw = dict(kw)
    ch = kw.pop("C", 4)
    src = o.lcg_image(sh, sw, ch, ti, seed=9)
    with lancir_plan(sw, sh, nw, nh, ch, ti, to, kw) as (L, pl, _):
        full = full_device(L, pl, upload(src), sw, sh, nw, nh, ch, to)
        for win in window_set(nw, nh, seed=12)[::2]:
            fi, n = query(L, pl, win)
            assert n == win[3] * fi.src_w * ch * 4
            sl, dl, d_src, d_dst, ws, _ = run_layout(L, pl, src, fi, n, win, to, layout)
            back = d_dst.cpu().numpy().view(to)
            assert cs.count_mismatch(crop(full, win), np.ascontiguousarray(dl.view(back))) == 0, win
            assert cs.guard_damage(dl, back) == 0, ("destination guard bytes overwritten", win)
            assert tail_damage(ws, n) == 0, ("store past lancirb200_window_workspace_bytes", win)
            assert np.array_equal(d_src.cpu().numpy(), sl.backing.view(np.uint8)), "source buffer written"


def route_failures():
    """(layout, kernels launched, kernels wanted) of each LANCIR layout whose window call runs other kernels
    than it is meant to cover; None when the profiler records no kernel activity."""
    routes = {"vec-in-vec-out": ["lancir_col4_kernel", "lancir_row4_kernel"],
              "scalar-in-vec-out": ["lancir_col_kernel", "lancir_row4_kernel"],
              "vec-in-scalar-out": ["lancir_col4_kernel", "lancir_row_kernel"],
              "scalar-in-scalar-out": ["lancir_col_kernel", "lancir_row_kernel"]}
    import torch
    sw, sh, nw, nh, ti, to, kw = LAYOUT_CASES[0]
    src = o.lcg_image(sh, sw, 4, ti, seed=9)
    win = (7, 5, 21, 11)
    failures = []
    with lancir_plan(sw, sh, nw, nh, 4, ti, to, kw) as (L, pl, _):
        fi, n = query(L, pl, win)
        assert fi.src_x0 % 2 == 1    # an odd footprint origin: pixel alignment comes from the buffer alone
        for layout, want in routes.items():
            *_, call = run_layout(L, pl, src, fi, n, win, to, layout)
            got = launched_kernels(call)
            if got is None:
                return None
            if got != want:
                failures.append((layout, got, want))
    torch.cuda.synchronize()
    return failures


def test_window_layouts_route_to_the_kernels_they_cover():
    """Run in a child process: a profiler session leaves state behind in the process that runs it, and the
    other routing tests of the suite profile in this one."""
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_lancir_window as t; "
            "print(json.dumps(t.route_failures()))" % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    failures = json.loads(r.stdout.strip().splitlines()[-1])
    if failures is None:
        pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
    assert not failures, failures


# ---- full size: 8K -> 4K RGBA u8 --------------------------------------------------------------------------

def test_full_size_windows():
    import torch
    sw, sh, nw, nh, ch = 7680, 4320, 3840, 2160, 4
    g = torch.Generator(device="cuda").manual_seed(5)
    d_src = torch.randint(0, 256, (sh * sw * ch,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, _):
        full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, u8)
        for win in [((nw - 1920) // 2 + 1, (nh - 1080) // 2 + 1, 1920, 1080), (3, 7, 1920, 1080),
                    (nw - 1921, nh - 1083, 1920, 1080), (777, 5, 1, 2000), (0, nh - 1, nw, 1),
                    (nw // 2 + 3, nh // 3 + 1, 17, 33), (nw - 1, 0, 1, nh)]:
            got = window_in_place(L, pl, d_src, sw, ch, u8, u8, win)
            assert cs.count_mismatch(crop(full, win), got) == 0, win
    del d_src
    torch.cuda.empty_cache()


# ---- the host form: the whole source in (pageable or page-locked), the window out --------------------------

@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("c", LAYOUT_CASES, ids=lambda c: "%dx%d-%dx%d-%s-%s-c%d" % (
    c[:4] + (np.dtype(c[4]).name, np.dtype(c[5]).name, c[6].get("C", 4))))
def test_window_host(c, pinned):
    import torch
    sw, sh, nw, nh, ti, to, kw = c
    kw = dict(kw)
    ch = kw.pop("C", 4)
    src = o.lcg_image(sh, sw, ch, ti, seed=10)
    sl = cs.source_layout(src, 6, 1, pinned=pinned)
    r, want = ab.CLancIR().resizeImage(src, nw, nh, ab.CLancIRParams(**kw), out_dtype=to)
    assert r == nh
    dev = torch.cuda.current_device()
    with lancir_plan(sw, sh, nw, nh, ch, ti, to, kw) as (L, pl, _):
        for win in window_set(nw, nh, seed=5)[::2]:
            # the C ABI
            dl = cs.guarded_dest((win[3], win[2], ch), to, 3, 1, pinned=pinned)
            es, eo = np.dtype(ti).itemsize, np.dtype(to).itemsize
            _ok(L.lancirb200_resize_window_host(pl, *win, sl.backing.ctypes.data + sl.origin * es, sl.pitch,
                                                dl.backing.ctypes.data + dl.origin * eo, dl.pitch))
            assert cs.count_mismatch(crop(want, win), np.ascontiguousarray(dl.view())) == 0, win
            assert cs.guard_damage(dl) == 0, win
            # the front-end, SrcSSize / NewSSize
            dl = cs.guarded_dest((win[3], win[2], ch), to, 5, 0, pinned=pinned)
            r, _ = ab.CLancIR().resizeImageWindow(sl.view(), nw, nh, *win,
                                                  ab.CLancIRParams(SrcSSize=sl.pitch, NewSSize=dl.pitch, **kw),
                                                  out_dtype=to, NewBuf=dl.view())
            assert r == win[3]
            assert cs.count_mismatch(crop(want, win), np.ascontiguousarray(dl.view())) == 0, win
            assert cs.guard_damage(dl) == 0, win
    assert torch.cuda.current_device() == dev


# ---- the front-end: Python and a C++ program --------------------------------------------------------------

@pytest.mark.parametrize("c", [(96, 54, 48, 27, 4, u8, u8, {}), (77, 51, 47, 29, 3, f32, u16, {"kx": 1.3, "ky": 2.2}),
                               (64, 48, 103, 77, 1, u16, f32, {"la": 4.0, "ox": 0.3})],
                         ids=lambda c: "%dx%d-%dx%d-c%d" % c[:5])
def test_front_end_windows(c):
    import torch
    sw, sh, nw, nh, ch, ti, to, kw = c
    src = o.lcg_image(sh, sw, ch, ti, seed=2)
    lr = ab.CLancIR()
    p = ab.CLancIRParams(**kw)
    r, want = lr.resizeImage(src, nw, nh, p, out_dtype=to)
    assert r == nh
    for win in window_set(nw, nh, seed=2)[::3]:
        r, got = lr.resizeImageWindow(src, nw, nh, *win, p, out_dtype=to)
        assert r == win[3] and cs.count_mismatch(crop(want, win), got) == 0, win
        fpn = lr.windowFootprint(src.shape, ti, nw, nh, to, win, p)
        n = lr.windowWorkspaceBytes(src.shape, ti, nw, nh, to, win, p)
        assert n == win[3] * fpn["src_w"] * ch * 4
        foot = np.ascontiguousarray(src[fpn["src_y0"]:fpn["src_y0"] + fpn["src_h"],
                                        fpn["src_x0"]:fpn["src_x0"] + fpn["src_w"]])
        d_src = upload(foot)
        d_dst = torch.empty(win[2] * win[3] * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
        ws = torch.empty(n, dtype=torch.uint8, device="cuda")
        assert lr.resizeImageWindowDevice(d_src.data_ptr(), src.shape, ti, d_dst.data_ptr(), nw, nh, to, win,
                                          ws.data_ptr(), p) == win[3]
        torch.cuda.synchronize()
        got = d_dst.cpu().numpy().view(to).reshape(win[3], win[2], ch)
        assert cs.count_mismatch(crop(want, win), got) == 0, win
    assert lr.resizeImageWindow(src, nw, nh, nw - 2, 0, 3, 1, p, out_dtype=to)[0] == 0
    assert lr.resizeImageWindow(src, nw, nh, 0, 0, 1, 1, p, out_dtype=to, NewBuf=None)[0] == 1


def test_user_window_program(tmp_path):
    ab.lib()
    exe = os.path.join(tempfile.mkdtemp(prefix="lancirb200_dropin_"), "user_window")
    libdir = os.path.join(ROOT, "avir_b200")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "dropin", "user_window.cpp"), "-L" + libdir, "-lavirb200",
                        "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    src = o.lcg_image(480, 640, 3, u8, seed=4)
    fin, fout = str(tmp_path / "in.bin"), str(tmp_path / "out.bin")
    src.tofile(fin)
    r = subprocess.run([exe, fout, fin], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    got = np.fromfile(fout, u8).reshape(129, 257, 3)
    rr, want = ab.CLancIR().resizeImage(src, 1024, 768)
    assert rr == 768
    assert cs.count_mismatch(crop(want, (301, 211, 257, 129)), got) == 0


# ---- a plan taller than one grid: the whole image is refused, its windows run -------------------------------

def test_tall_plan_windows():
    import torch
    sw, sh, nw, nh, ch = 6, 35000, 4, 70001, 1
    src = o.lcg_image(sh, sw, ch, u8, seed=6)
    with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, dp):
        want = np.zeros((nh, nw, ch), u8)
        assert cs.port().lancir_port_resize(dp, src.ctypes.data, sw * ch, want.ctypes.data, nw * ch) == 0
        d_src = upload(src)
        n = C.c_size_t()
        _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
        buf = torch.empty(max(n.value, nh * nw * ch), dtype=torch.uint8, device="cuda")
        assert L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, buf.data_ptr(), nw * ch, buf.data_ptr(),
                                          None) == ERR_UNSUPPORTED
        for win in [(0, 0, nw, 65535), (1, nh - 65535, 2, 65535), (3, 40000, 1, 7), (0, nh - 1, nw, 1)]:
            got = window_in_place(L, pl, d_src, sw, ch, u8, u8, win)
            assert cs.count_mismatch(crop(want, win), got) == 0, win
        fi, wn = query(L, pl, (0, 0, nw, 65536))
        assert L.lancirb200_resize_window_device(pl, 0, 0, nw, 65536, d_src.data_ptr(), sw * ch, buf.data_ptr(),
                                                 nw * ch, buf.data_ptr(), None) == ERR_UNSUPPORTED
    torch.cuda.synchronize()


# ---- errors ------------------------------------------------------------------------------------------------

def test_window_errors():
    import torch
    d = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    h_buf = np.zeros(1 << 20, np.uint8)
    p = d.data_ptr()
    with lancir_plan(96, 54, 48, 27, 4, u8, u8, {}) as (L, pl, _):
        for win in [(0, 0, 0, 1), (-1, 0, 4, 4), (45, 0, 4, 4), (0, 24, 4, 4), (2 ** 31 - 1, 0, 2, 1),
                    (0, 2 ** 31 - 1, 1, 2)]:
            fi, n = LancirWindowInfo(), C.c_size_t()
            assert L.lancirb200_window_query(pl, *win, C.byref(fi)) == ERR_BAD_ARG, win
            assert L.lancirb200_window_workspace_bytes(pl, *win, C.byref(n)) == ERR_BAD_ARG, win
            assert L.lancirb200_resize_window_device(pl, *win, p, 384, p, 192, p, None) == ERR_BAD_ARG, win
            assert L.lancirb200_resize_window_host(pl, *win, h_buf.ctypes.data, 384, h_buf.ctypes.data,
                                                   192) == ERR_BAD_ARG, win
        fi, n = query(L, pl, (10, 10, 20, 10))
        assert L.lancirb200_resize_window_device(pl, 10, 10, 20, 10, p, fi.src_w * 4 - 1, p, 80, p,
                                                 None) == ERR_BAD_ARG
        assert L.lancirb200_resize_window_device(pl, 10, 10, 20, 10, p, fi.src_w * 4, p, 79, p, None) == ERR_BAD_ARG
    torch.cuda.synchronize()


# ---- value-domain sources ----------------------------------------------------------------------------------

VALUE_CASES = [(96, 64, 48, 32, 4, u8), (96, 64, 48, 32, 4, f32), (64, 48, 103, 77, 4, u16),
               (77, 51, 47, 29, 3, u8), (77, 51, 47, 29, 1, u16), (77, 51, 47, 29, 2, f32)]


@pytest.mark.parametrize("kind", ("range", "huge", "nonfinite", "tiny", "ties"))
@pytest.mark.parametrize("c", VALUE_CASES, ids=_tid)
def test_window_value_domain(c, kind):
    sw, sh, nw, nh, ch, to = c
    src = cs.value_image((0, sw, sh, nw, nh, ch, f32, to, 8, {}), kind)
    ref = None
    if o.have_ref():
        r, ref = o.lancir_ref(src, nw, nh, to)
        assert r == nh
    check_windows(src, nw, nh, to, {}, window_set(nw, nh, seed=7), mismatch=cs.value_mismatch, ref=ref)
