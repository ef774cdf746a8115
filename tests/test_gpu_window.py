"""Destination windows on the GPU (run with -m gpu on an H100): avirb200_resize_window_device /
_host and the front-end's resizeImageWindow* against the whole image.

A window (x0, y0, w, h) must equal the same pixels of avirb200_resize_device on the whole image
(and of upstream's output where oracle/_ref is present), on every kernel family, for every small
case, with the source buffer holding exactly the window's footprint.  Buffer layouts follow
test_gpu_layouts.py: poisoned source guards, sentinel destination guards and a sentinel tail behind
the workspace the library asked for."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_gpu_layouts import (F, FAMILIES, G, N, S, TILE, W, _ok, avir_plan, guarded_workspace, launched_kernels,
                              lib, plan_workspace, tail_damage)
from test_window import WindowInfo, crop, window_set

pytestmark = pytest.mark.gpu

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
ERR_BAD_ARG, ERR_UNSUPPORTED = -1, -4


def wlib():
    L = lib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    L.avirb200_window_query.argtypes = [vp, i, i, i, i, vp]
    L.avirb200_window_workspace_bytes.argtypes = [vp, i, i, i, i, vp]
    L.avirb200_resize_window_device.argtypes = [vp, i, i, i, i, vp, sz, vp, sz, vp, vp]
    L.avirb200_resize_window_host.argtypes = [vp, i, i, i, i, vp, sz, vp, sz]
    return L


def query(L, pl, win):
    fi, n = WindowInfo(), C.c_size_t()
    _ok(L.avirb200_window_query(pl, *win, C.byref(fi)))
    _ok(L.avirb200_window_workspace_bytes(pl, *win, C.byref(n)))
    return fi, n.value


def _is_errd(case):
    return case[0] >= 3 and np.dtype(case[7]).kind != "f"


def full_device(L, pl, case, d_src):
    """avirb200_resize_device on the whole image (packed buffers)."""
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    n = plan_workspace(L, pl)
    d_dst = torch.empty(nh * nw * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    _ok(L.avirb200_resize_device(pl, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch, ws.data_ptr(), None))
    torch.cuda.synchronize()
    return d_dst.cpu().numpy().view(to).reshape(nh, nw, ch)


def window_in_place(L, pl, case, d_src, win):
    """The window with d_src pointing at its footprint inside the whole device image (pitched)."""
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    fi, n = query(L, pl, win)
    es = np.dtype(ti).itemsize
    d_dst = torch.empty(win[2] * win[3] * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
    ws = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
    src_ptr = d_src.data_ptr() + (fi.src_y0 * sw + fi.src_x0) * ch * es
    _ok(L.avirb200_resize_window_device(pl, *win, src_ptr, sw * ch, d_dst.data_ptr(), win[2] * ch, ws.data_ptr(),
                                        None))
    torch.cuda.synchronize()
    return d_dst.cpu().numpy().view(to).reshape(win[3], win[2], ch)


def upload(img):
    import torch
    return torch.from_numpy(np.ascontiguousarray(img).view(np.uint8).reshape(-1)).cuda()


# ---- equality with the whole image: every small case x every kernel family x the window set --------------

@FAMILIES
@pytest.mark.parametrize("case", [c for c in cs.SMALL_CASES if not _is_errd(c)], ids=cs.case_id)
def test_window_equals_the_whole_image(case, family):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    ref = cs.ref_output(case, src) if o.have_ref() else None
    with avir_plan(case, family) as (_, pl):
        L = wlib()
        d_src = upload(src)
        full = full_device(L, pl, case, d_src)
        if ref is not None:
            assert cs.count_mismatch(ref, full) == 0
        for win in window_set(nw, nh, seed=family):
            got = window_in_place(L, pl, case, d_src, win)
            assert cs.count_mismatch(crop(full, win), got) == 0, win


@pytest.mark.parametrize("kind", ("range", "huge", "nonfinite", "tiny"))
@pytest.mark.parametrize("case", [(0, 256, 192, 128, 96, 4, f32, u8, 8, {"buildmode": 1}),
                                  (2, 256, 192, 64, 48, 4, f32, u16, 16, {"buildmode": 1}),
                                  (1, 256, 192, 64, 48, 4, f32, f32, 16, {"buildmode": 0}),
                                  (1, 150, 90, 100, 55, 4, f32, u16, 16, {})], ids=cs.case_id)
def test_window_value_domain(case, kind):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.value_image(case, kind)
    with avir_plan(case, 0) as (_, pl):
        L = wlib()
        d_src = upload(src)
        full = full_device(L, pl, case, d_src)
        for win in window_set(nw, nh, seed=7)[::2]:
            got = window_in_place(L, pl, case, d_src, win)
            assert cs.value_mismatch(crop(full, win), got) == 0, win


# ---- buffer layouts: the footprint alone inside poisoned guards, guarded destination and workspace ----------

LAYOUT_CASES = [(2, 192, 108, 96, 54, 4, f32, f32, 16, {}), (1, 256, 256, 64, 64, 4, u16, u16, 16, {}),
                (2, 384, 216, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),
                (1, 240, 135, 480, 270, 4, u8, u8, 8, {}), TILE,
                (0, 320, 240, 160, 120, 3, u8, u8, 8, {}), (1, 192, 108, 96, 54, 1, f32, f32, 16, {}),
                (1, 192, 108, 96, 54, 4, f64, f64, 16, {}), (0, 120, 80, 60, 40, 3, f32, f64, 16, {"gamma": True})]


def footprint_layout(img, fi, extra_pitch, elem_offset):
    """The footprint of `img` alone in a buffer: two poisoned guard rows above and below, poisoned
    row padding; every element outside the footprint is cs.poison_of(dtype)."""
    ch = img.shape[2]
    pitch = fi.src_w * ch + extra_pitch
    back = cs.host_array((fi.src_h + 4) * pitch + elem_offset + 8, img.dtype)
    back[:] = cs.poison_of(img.dtype)
    lay = cs.Layout(back, 2 * pitch + elem_offset, pitch, (fi.src_h, fi.src_w, ch))
    lay.view()[:] = img[fi.src_y0:fi.src_y0 + fi.src_h, fi.src_x0:fi.src_x0 + fi.src_w]
    return lay


@FAMILIES
@pytest.mark.parametrize("pads", [(0, 0, 0, 0), (8, 0, 2, 0), (5, 1, 3, 1)], ids=["packed", "padded", "odd"])
@pytest.mark.parametrize("case", LAYOUT_CASES, ids=cs.case_id)
def test_window_buffer_layouts(case, pads, family):
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    sx, so, dx, do = pads
    src = cs.make_input(case)
    with avir_plan(case, family) as (_, pl):
        L = wlib()
        full = full_device(L, pl, case, upload(src))
        for win in window_set(nw, nh, seed=11)[::3]:
            fi, n = query(L, pl, win)
            sl = footprint_layout(src, fi, sx, so)
            dl = cs.guarded_dest((win[3], win[2], ch), to, dx, do)
            d_src, d_dst, ws = upload(sl.backing), upload(dl.backing), guarded_workspace(n)
            es, eo = np.dtype(ti).itemsize, np.dtype(to).itemsize
            _ok(L.avirb200_resize_window_device(pl, *win, d_src.data_ptr() + sl.origin * es, sl.pitch,
                                                d_dst.data_ptr() + dl.origin * eo, dl.pitch, ws.data_ptr(), None))
            torch.cuda.synchronize()
            back = d_dst.cpu().numpy().view(to)
            assert cs.count_mismatch(crop(full, win), np.ascontiguousarray(dl.view(back))) == 0, win
            assert cs.guard_damage(dl, back) == 0, ("destination guard bytes overwritten", win)
            assert tail_damage(ws, n) == 0, ("store past avirb200_window_workspace_bytes", win)
            assert np.array_equal(d_src.cpu().numpy(), sl.backing.view(np.uint8)), "source buffer written"


# ---- larger inputs: full-size cfg3 and cfg4 windows at odd offsets ------------------------------------------

@pytest.mark.parametrize("case", [(2, 7680, 4320, 3840, 2160, 4, f32, f32, 16, {}),
                                  (1, 16384, 16384, 4096, 4096, 4, u16, u16, 16, {})], ids=["cfg3", "cfg4"])
def test_full_size_windows(case):
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    g = torch.Generator(device="cuda").manual_seed(5)
    if ti == f32:
        d_src = torch.rand(sh * sw * ch, generator=g, device="cuda", dtype=torch.float32).view(torch.uint8)
    else:
        d_src = torch.randint(0, 65536, (sh * sw * ch,), generator=g, device="cuda", dtype=torch.int32)
        d_src = d_src.to(torch.uint16).view(torch.uint8)
    with avir_plan(case, 0) as (_, pl):
        L = wlib()
        full = full_device(L, pl, case, d_src)
        for win in [(nw // 4 + 1, nh // 5 + 3, 1920, 1080), (3, 7, 1920, 1080), (nw - 1921, nh - 1083, 1920, 1080),
                    (777, 5, 1, 2000), (0, nh - 1, nw, 1), (nw // 2 + 3, nh // 3 + 1, 17, 33)]:
            got = window_in_place(L, pl, case, d_src, win)
            assert cs.count_mismatch(crop(full, win), got) == 0, win
    del d_src
    torch.cuda.empty_cache()


# ---- the host form: the whole source in (pageable or page-locked), the window out ---------------------------

@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("case", LAYOUT_CASES[:2] + LAYOUT_CASES[5:8], ids=cs.case_id)
def test_window_host(case, pinned):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    sl = cs.source_layout(src, 6, 1, pinned=pinned)
    with avir_plan(case, 0) as (_, pl):
        L = wlib()
        full = full_device(L, pl, case, upload(src))
        for win in window_set(nw, nh, seed=5)[::3]:
            dl = cs.guarded_dest((win[3], win[2], ch), to, 3, 1, pinned=pinned)
            es, eo = np.dtype(ti).itemsize, np.dtype(to).itemsize
            _ok(L.avirb200_resize_window_host(pl, *win, sl.backing.ctypes.data + sl.origin * es, sl.pitch,
                                              dl.backing.ctypes.data + dl.origin * eo, dl.pitch))
            assert cs.count_mismatch(crop(full, win), np.ascontiguousarray(dl.view())) == 0, win
            assert cs.guard_damage(dl) == 0, win


# ---- the front-end: resizeImageWindow / resizeImageWindowDevice share the resize's cached plan --------------

@pytest.mark.parametrize("case", [(2, 192, 108, 96, 54, 4, f32, f32, 16, {}),
                                  (1, 100, 60, 150, 77, 4, u8, u8, 8, {}),
                                  (0, 120, 80, 60, 40, 3, u8, f64, 8, {"gamma": True})], ids=cs.case_id)
def test_front_end_windows(case):
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case)
    want = cs.gpu_output(case, src)
    rs, v = cs.resizer_and_vars(case)
    for win in window_set(nw, nh, seed=2)[::4]:
        got = rs.resizeImageWindow(src, nw, nh, win, 0.0, v, out_dtype=to)
        assert cs.count_mismatch(crop(want, win), got) == 0, win
        fpn = rs.windowFootprint(src.shape, ti, nw, nh, to, win, 0.0, v)
        n = rs.windowWorkspaceBytes(src.shape, ti, nw, nh, to, win, 0.0, v)
        foot = np.ascontiguousarray(src[fpn["src_y0"]:fpn["src_y0"] + fpn["src_h"],
                                        fpn["src_x0"]:fpn["src_x0"] + fpn["src_w"]])
        d_src = upload(foot)
        d_dst = torch.empty(win[2] * win[3] * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
        ws = torch.empty(max(n, 1), dtype=torch.uint8, device="cuda")
        rs.resizeImageWindowDevice(d_src.data_ptr(), src.shape, ti, d_dst.data_ptr(), nw, nh, to, win, ws.data_ptr(),
                                   0.0, v)
        torch.cuda.synchronize()
        got = d_dst.cpu().numpy().view(to).reshape(win[3], win[2], ch)
        assert cs.count_mismatch(crop(want, win), got) == 0, win
    with pytest.raises(ab.AvirB200Error):
        rs.resizeImageWindow(src, nw, nh, (nw - 2, 0, 3, 1), 0.0, v, out_dtype=to)


# ---- errors -------------------------------------------------------------------------------------------------

def test_window_errors():
    import torch
    d = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    h_buf = np.zeros(1 << 20, np.uint8)
    p = d.data_ptr()
    ERRD = (4, 120, 80, 60, 40, 4, u8, u8, 8, {})
    with avir_plan(ERRD, 0) as (_, pl):
        L = wlib()
        fi, n = WindowInfo(), C.c_size_t()
        assert L.avirb200_window_query(pl, 1, 2, 10, 10, C.byref(fi)) == ERR_UNSUPPORTED
        assert L.avirb200_window_workspace_bytes(pl, 1, 2, 10, 10, C.byref(n)) == ERR_UNSUPPORTED
        assert L.avirb200_resize_window_device(pl, 1, 2, 10, 10, p, 480, p, 40, p, None) == ERR_UNSUPPORTED
        assert L.avirb200_resize_window_host(pl, 1, 2, 10, 10, h_buf.ctypes.data, 480, h_buf.ctypes.data,
                                             40) == ERR_UNSUPPORTED
    CFG3 = (2, 192, 108, 96, 54, 4, f32, f32, 16, {})
    with avir_plan(CFG3, 0) as (_, pl):
        L = wlib()
        for win in [(0, 0, 0, 1), (-1, 0, 4, 4), (93, 0, 4, 4), (0, 51, 4, 4), (2 ** 31 - 1, 0, 2, 1),
                    (0, 2 ** 31 - 1, 1, 2)]:
            fi, n = WindowInfo(), C.c_size_t()
            assert L.avirb200_window_query(pl, *win, C.byref(fi)) == ERR_BAD_ARG, win
            assert L.avirb200_window_workspace_bytes(pl, *win, C.byref(n)) == ERR_BAD_ARG, win
            assert L.avirb200_resize_window_device(pl, *win, p, 768, p, 384, p, None) == ERR_BAD_ARG, win
            assert L.avirb200_resize_window_host(pl, *win, h_buf.ctypes.data, 768, h_buf.ctypes.data,
                                                 384) == ERR_BAD_ARG, win
        # a source pitch narrower than the footprint's rows
        fi, n = query(L, pl, (10, 10, 20, 20))
        assert L.avirb200_resize_window_device(pl, 10, 10, 20, 20, p, fi.src_w * 4 - 1, p, 80, p,
                                               None) == ERR_BAD_ARG
    torch.cuda.synchronize()


# ---- routing: a window of a headline chain runs on the streaming kernels --------------------------------------

WINDOW_ROUTES = [
    # (case, kernel family, window, kernels launched in order)
    ((2, 192, 108, 96, 54, 4, f32, f32, 16, {}), 0, (5, 3, 60, 40), [S, S]),          # cfg3 chain (DIL)
    ((1, 192, 108, 96, 54, 4, f32, f32, 16, {}), 0, (17, 9, 31, 20), [S, S]),         # cfg3 chain (float4)
    ((1, 256, 256, 64, 64, 4, u16, u16, 16, {}), 0, (1, 2, 40, 30), [S, S]),          # cfg4 chain
    ((2, 192, 108, 96, 54, 4, f32, f32, 16, {}), 2, (5, 3, 60, 40), [F, F]),
    (TILE, 0, (3, 4, 50, 20), [F, F]),
    ((2, 192, 108, 96, 54, 4, f32, f32, 16, {}), 1, (5, 3, 60, 40), [G, G]),
    ((0, 320, 240, 160, 120, 3, u8, u8, 8, {}), 2, (7, 5, 33, 21), [W, F, F, N]),
]


def test_windows_route_to_the_kernels_they_cover():
    import torch
    failures = []
    for case, family, win, want in WINDOW_ROUTES:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        src = cs.make_input(case)
        with avir_plan(case, family) as (_, pl):
            L = wlib()
            d_src = upload(src)
            window_in_place(L, pl, case, d_src, win)  # (tables built, kernels loaded)
            got = launched_kernels(lambda: window_in_place(L, pl, case, d_src, win))
        if got is None:
            pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
        if got != want:
            failures.append((cs.case_id(case), family, win, got, want))
    torch.cuda.synchronize()
    assert not failures, failures
