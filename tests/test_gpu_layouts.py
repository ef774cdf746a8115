"""Caller buffer layouts on the GPU (run with -m gpu on an H100): padded and odd pitches, bases offset
by one element, page-locked and pageable host memory, on every entry point and kernel family.

The engine picks its kernel from the caller's layout: the streaming and tile kernels need pixel-
aligned rows (source pitch % 4 == 0, destination pitch % 2 == 0, aligned bases), anything else runs
the generic kernel, per pass; LANCIR picks its 4-channel vector kernels per pass the same way.  So
every layout below is a different kernel mix, and each must give upstream's bits:

* sources are padded with poison (NaN, or the type's maximum) -- a read past a row end that reaches
  a result shows up as a mismatch;
* destinations carry guard rows and pitch padding filled with a sentinel byte, and the workspace a
  64 KiB sentinel tail past the size the library asked for -- a stray store shows up as damage;
* the reference is upstream on the same padded source (its SrcScanlineSize / SrcSSize / NewSSize),
  or the C port on the packed image where oracle/_ref is absent; 0 mismatching elements.

test_layouts_route_to_the_kernels_they_cover records the launched kernels with torch.profiler, so
that a later change to the routing predicates cannot quietly turn these into contiguous-layout tests.
"""
import contextlib
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o

pytestmark = pytest.mark.gpu

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TAIL = 64 << 10  # workspace guard bytes past what the library asked for
FAMILIES = pytest.mark.parametrize("family", [0, 2, 1], ids=["product", "tile", "generic"])

# small images over the chains, types and channel counts whose kernels differ
CFG3_DIL = (2, 192, 108, 96, 54, 4, f32, f32, 16, {})
CFG3_F4 = (1, 192, 108, 96, 54, 4, f32, f32, 16, {})
CFG4 = (1, 256, 256, 64, 64, 4, u16, u16, 16, {})
CFG5 = (2, 384, 216, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3})
CFG2 = (1, 240, 135, 480, 270, 4, u8, u8, 8, {})
TILE = (1, 150, 90, 100, 55, 4, u8, u8, 8, {})            # non-integer ratio: tile kernel
RGB = (0, 320, 240, 160, 120, 3, u8, u8, 8, {})           # widened onto the 4-channel kernels
GRAY = (1, 192, 108, 96, 54, 1, f32, f32, 16, {})         # widened, one channel
F64 = (1, 192, 108, 96, 54, 4, f64, f64, 16, {})          # narrow_f64_kernel / widen_f32_kernel
ERRD = (4, 120, 80, 60, 40, 4, u8, u8, 8, {})             # errd_kernel stores with the caller's pitch
DEVICE_CASES = [CFG3_DIL, CFG3_F4, CFG4, CFG5, CFG2, TILE, RGB, GRAY, F64, ERRD]
WIDENED = [RGB, GRAY]


def _src_pitch(row, kind):
    p = row + 5
    p += (-p) % 4
    return {"pad4": p, "padodd": p + 1}[kind]            # pitch % 4 == 0 / == 1


def _dst_pitch(row, kind):
    p = row + 3
    return {"pad2": p + p % 2, "odd": p + 1 - p % 2}[kind]  # even / odd


# name: (source pitch kind, source element offset, destination pitch kind, destination element offset)
LAYOUTS = {
    "L0-packed": (None, 0, None, 0),
    "L1-src-pad4": ("pad4", 0, None, 0),
    "L2-src-pitch-not4": ("padodd", 0, None, 0),
    "L3-src-offset1": (None, 1, None, 0),
    "L4-dst-pad2": (None, 0, "pad2", 0),
    "L5-dst-odd": (None, 0, "odd", 0),
    "L5-dst-offset1": (None, 0, None, 1),
    "L6-src-offset1-dst-pad2": (None, 1, "pad2", 0),
    "L6-src-pad4-dst-odd": ("pad4", 0, "odd", 0),
}


def make_layouts(case, layout, seed=3, pinned=False):
    """(source Layout holding the case's input, guarded destination Layout)."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    sk, so, dk, do = LAYOUTS[layout]
    src = cs.make_input(case, seed=seed)
    sx = _src_pitch(sw * ch, sk) - sw * ch if sk else 0
    dx = _dst_pitch(nw * ch, dk) - nw * ch if dk else 0
    return (cs.source_layout(src, sx, so, pinned=pinned),
            cs.guarded_dest((nh, nw, ch), to, dx, do, pinned=pinned))


def expected(case, sl):
    """Upstream on the same padded source (SrcScanlineSize = its pitch), else the port."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    if o.have_ref():
        return o.ref_resize(sl.view(), nw, nh, to, fpclass=fp, resbits=rb, src_pitch=sl.pitch,
                            **cs.ref_kwargs(kw))
    return cs.port_output(case, np.ascontiguousarray(sl.view()))[0]


def lib():
    L = ab.lib()
    vp, sz = C.c_void_p, C.c_size_t
    L.avirb200_plan_set_option.argtypes = [vp, C.c_int, C.c_int]
    L.avirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    L.avirb200_row_pass_device.argtypes = [vp, vp, sz, vp, vp]
    L.avirb200_col_pass_device.argtypes = [vp, vp, vp, sz, vp]
    L.avirb200_resize_device_batch.argtypes = [vp, C.c_int, vp, sz, vp, sz, vp, vp]
    L.avirb200_resize_sharded_local.argtypes = [vp, C.c_int, vp, sz, vp, sz, vp, vp]
    L.avirb200_resize_host.argtypes = [vp, vp, sz, vp, sz]
    L.lancirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    return L


def _ok(r):
    assert r == 0, ab.lib().avirb200_last_error().decode()


@contextlib.contextmanager
def avir_plan(case, family=0, options=None):
    """A C-ABI plan of the case, as CImageResizer<>::resizeImage builds it, with plan options set."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, kw.get("k", 0.0), v)
    L, pl = lib(), C.c_void_p()
    try:
        _ok(L.avirb200_plan_create(C.c_void_p(dp), C.byref(pl)))
        _ok(L.avirb200_plan_set_option(pl, ab.OPT_KERNEL_FAMILY, family))
        for opt, val in (options or {}).items():
            _ok(L.avirb200_plan_set_option(pl, opt, val))
        yield L, pl
    finally:
        if pl.value:
            L.avirb200_plan_destroy(pl)
        rs.free_descriptor(h)


def plan_workspace(L, pl):
    b = C.c_size_t()
    _ok(L.avirb200_plan_workspace_bytes(pl, C.byref(b)))
    return b.value


def to_device(lay):
    import torch
    return torch.from_numpy(np.ascontiguousarray(lay.backing).view(np.uint8)).cuda()


def dptr(t, lay):
    return t.data_ptr() + lay.origin * lay.backing.dtype.itemsize


def guarded_workspace(nbytes):
    import torch
    return torch.full((nbytes + TAIL,), cs.SENTINEL, dtype=torch.uint8, device="cuda")


def tail_damage(ws, nbytes):
    return int((ws[nbytes:] != cs.SENTINEL).sum().item())


def check(want, dl, d_dst, what=""):
    """0 mismatching elements in the destination image, every guard byte intact."""
    import torch
    torch.cuda.synchronize()
    back = d_dst.cpu().numpy().view(dl.backing.dtype)
    got = np.ascontiguousarray(dl.view(back))
    assert cs.count_mismatch(want, got) == 0, what
    assert cs.guard_damage(dl, back) == 0, "destination guard bytes overwritten " + what


# ---- avirb200_resize_device: every layout x every kernel family --------------------------------------

@FAMILIES
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("case", DEVICE_CASES, ids=cs.case_id)
def test_resize_device_layouts(case, layout, family):
    sl, dl = make_layouts(case, layout)
    want = expected(case, sl)
    with avir_plan(case, family) as (L, pl):
        n = plan_workspace(L, pl)
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
        _ok(L.avirb200_resize_device(pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch,
                                     ws.data_ptr(), None))
        check(want, dl, d_dst)
        assert tail_damage(ws, n) == 0, "store past avirb200_plan_workspace_bytes"
        assert np.array_equal(d_src.cpu().numpy(), sl.backing.view(np.uint8)), "source buffer written"


def test_widened_cases_are_widened():
    """The 1- and 3-channel cases run on the 4-channel kernels (their intermediate is 4 floats a
    pixel), so that they cover the widened plans' layout."""
    for case in WIDENED:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        with avir_plan(case) as (L, pl):
            assert plan_workspace(L, pl) >= nw * sh * 4 * 4, cs.case_id(case)


# ---- the two passes called one by one ---------------------------------------------------------------

SPLIT_LAYOUTS = ["L0-packed", "L2-src-pitch-not4", "L5-dst-odd", "L6-src-offset1-dst-pad2", "L6-src-pad4-dst-odd"]


@FAMILIES
@pytest.mark.parametrize("layout", SPLIT_LAYOUTS)
@pytest.mark.parametrize("case", [CFG3_DIL, CFG4, CFG5, TILE, RGB, GRAY], ids=cs.case_id)
def test_split_passes_layouts(case, layout, family):
    """avirb200_row_pass_device then avirb200_col_pass_device = avirb200_resize_device."""
    sl, dl = make_layouts(case, layout, seed=4)
    want = expected(case, sl)
    with avir_plan(case, family) as (L, pl):
        n = plan_workspace(L, pl)
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
        _ok(L.avirb200_row_pass_device(pl, dptr(d_src, sl), sl.pitch, ws.data_ptr(), None))
        _ok(L.avirb200_col_pass_device(pl, ws.data_ptr(), dptr(d_dst, dl), dl.pitch, None))
        check(want, dl, d_dst)
        assert tail_damage(ws, n) == 0


# ---- a batch whose frames sit at different alignments ----------------------------------------------

@FAMILIES
@pytest.mark.parametrize("case", [CFG3_DIL, CFG4, TILE, RGB], ids=cs.case_id)
def test_batch_frames_at_mixed_alignments(case, family):
    """avirb200_resize_device_batch routes every frame by its own pointers: frames whose bases are
    one to three elements off the pixel alignment run other kernels than their neighbours."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    n = 4
    spitch = _src_pitch(sw * ch, "pad4")
    dpitch = _dst_pitch(nw * ch, "pad2")
    sls = [cs.source_layout(cs.make_input(case, seed=70 + i), spitch - sw * ch, i) for i in range(n)]
    dls = [cs.guarded_dest((nh, nw, ch), to, dpitch - nw * ch, i % 2) for i in range(n)]
    with avir_plan(case, family) as (L, pl):
        nb = plan_workspace(L, pl)
        d_srcs, d_dsts, ws = [to_device(s) for s in sls], [to_device(d) for d in dls], guarded_workspace(nb)
        sp = (C.c_void_p * n)(*[dptr(t, s) for t, s in zip(d_srcs, sls)])
        dp = (C.c_void_p * n)(*[dptr(t, d) for t, d in zip(d_dsts, dls)])
        _ok(L.avirb200_resize_device_batch(pl, n, sp, spitch, dp, dpitch, ws.data_ptr(), None))
        for i in range(n):
            check(expected(case, sls[i]), dls[i], d_dsts[i], "frame %d" % i)
        assert tail_damage(ws, nb) == 0


# ---- the sharded schedule on one device ---------------------------------------------------------

SHARD_CASES = [
    (2, 192, 216, 96, 108, 4, f32, f32, 16, {}),                            # headline chain
    (1, 256, 384, 64, 96, 4, u16, u16, 16, {}),                             # cfg4 chain
    (0, 320, 360, 160, 180, 3, u8, u8, 8, {}),                              # widened RGB
    (1, 192, 216, 96, 108, 1, f32, f32, 16, {}),                            # widened gray
]


@FAMILIES
@pytest.mark.parametrize("overlap", [3, 1])
@pytest.mark.parametrize("nranks", [2, 3, 5])
@pytest.mark.parametrize("layout", ["L0-packed", "L1-src-pad4", "L4-dst-pad2", "L3-src-offset1"])
@pytest.mark.parametrize("case", SHARD_CASES, ids=cs.case_id)
def test_sharded_local_layouts(case, layout, nranks, overlap, family):
    sl, dl = make_layouts(case, layout, seed=5)
    want = expected(case, sl)
    with avir_plan(case, family, {ab.OPT_OVERLAP_HALO: overlap}) as (L, pl):
        n = 0
        for r in range(nranks):
            b = C.c_size_t()
            _ok(L.avirb200_shard_workspace_bytes(pl, r, nranks, C.byref(b)))
            n += b.value
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
        _ok(L.avirb200_resize_sharded_local(pl, nranks, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch,
                                            ws.data_ptr(), None))
        check(want, dl, d_dst)
        assert tail_damage(ws, n) == 0, "store past the shards' workspace"


# ---- host calls: padded SrcScanlineSize, pageable and page-locked memory, row bands ----------------

HOST_CASES = [CFG3_DIL, CFG4, RGB, GRAY, TILE]
MEMS = {"pageable": (False, False), "pinned": (True, True), "pinned-src": (True, False), "pinned-dst": (False, True)}


@pytest.fixture(params=[0, 2, 1], ids=["product", "tile", "generic"])
def host_family(request):
    ab.set_option(ab.OPT_KERNEL_FAMILY, request.param)
    yield request.param
    ab.set_option(ab.OPT_KERNEL_FAMILY, -1)


@pytest.mark.parametrize("bands", [1, 2, 7])
@pytest.mark.parametrize("mem", list(MEMS))
@pytest.mark.parametrize("case", HOST_CASES, ids=cs.case_id)
def test_host_call_padded_source(case, mem, bands, host_family):
    """CImageResizer<>::resizeImage with SrcScanlineSize > row length, unbanded and cut into row
    bands (the pipelined form: page-locked buffers are copied directly, pageable ones through the
    library's bounce buffers with the caller's pitch)."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    pin_src, pin_dst = MEMS[mem]
    sl = cs.source_layout(cs.make_input(case, seed=6), _src_pitch(sw * ch, "padodd") - sw * ch, 0, pinned=pin_src)
    dl = cs.guarded_dest((nh, nw, ch), to, pinned=pin_dst)
    want = expected(case, sl)
    rs, v = cs.resizer_and_vars(case)
    ab.set_option(ab.OPT_HOST_BANDS, bands)
    try:
        rs.resizeImage(sl.view(), nw, nh, kw.get("k", 0.0), v, out_dtype=to, NewBuf=dl.view(),
                       SrcScanlineSize=sl.pitch)
    finally:
        ab.set_option(ab.OPT_HOST_BANDS, -1)
    assert cs.count_mismatch(want, np.ascontiguousarray(dl.view())) == 0
    assert cs.guard_damage(dl) == 0


@pytest.mark.parametrize("bands", [1, 3])
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("case", [CFG3_DIL, RGB, F64], ids=cs.case_id)
def test_host_c_abi_padded_destination(case, pinned, bands):
    """avirb200_resize_host with padded source AND destination pitches (the C ABI takes both)."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    sl = cs.source_layout(cs.make_input(case, seed=8), _src_pitch(sw * ch, "pad4") - sw * ch, pinned=pinned)
    dl = cs.guarded_dest((nh, nw, ch), to, _dst_pitch(nw * ch, "odd") - nw * ch, pinned=pinned)
    want = expected(case, sl)
    with avir_plan(case, 0, {ab.OPT_HOST_BANDS: bands}) as (L, pl):
        _ok(L.avirb200_resize_host(pl, sl.view().ctypes.data, sl.pitch, dl.view().ctypes.data, dl.pitch))
    assert cs.count_mismatch(want, np.ascontiguousarray(dl.view())) == 0
    assert cs.guard_damage(dl) == 0


# ---- LANCIR ------------------------------------------------------------------------------------

LANCIR_CASES = [
    (96, 54, 48, 27, u8, u8, {}),                    # k = 2: 12 taps
    (64, 48, 103, 77, u8, u8, {}),                   # upsizing: 6 taps
    (64, 64, 16, 16, u16, u16, {}),                  # k = 4: 24 taps
    (50, 30, 33, 17, f32, u8, {}),                   # other kernel lengths
    (77, 51, 47, 29, f32, f32, {"C": 3, "kx": 1.3, "ky": 2.2}),
    (96, 54, 48, 27, u8, f32, {"C": 1}),
]


def _lancir_id(c):
    sw, sh, nw, nh, ti, to, kw = c
    return "%dx%d-%dx%d-%s-%s-c%d" % (sw, sh, nw, nh, np.dtype(ti).name, np.dtype(to).name, kw.get("C", 4))


# (source pitch kind, source offset, destination pitch % 4, destination offset): which LANCIR kernels
# a 4-channel image takes -- vector column pass (lancir_col4_kernel) needs a pixel-aligned source,
# vector row pass (lancir_row4_kernel) a pixel-aligned destination
LANCIR_LAYOUTS = {
    "vec-in-vec-out": ("pad4", 0, 0, 0),
    "scalar-in-vec-out": ("pad4", 1, 0, 0),
    "vec-in-scalar-out": ("pad4", 0, 2, 0),
    "scalar-in-scalar-out": ("padodd", 0, 0, 1),
}


def lancir_layouts(c, layout, seed=9):
    sw, sh, nw, nh, ti, to, kw = c
    ch = kw.get("C", 4)
    sk, so, dmod, do = LANCIR_LAYOUTS[layout]
    src = o.lcg_image(sh, sw, ch, ti, seed=seed)
    p = nw * ch + 4
    p += (dmod - p) % 4
    sl = cs.source_layout(src, _src_pitch(sw * ch, sk) - sw * ch, so)
    return sl, (lambda: cs.guarded_dest((nh, nw, ch), to, p - nw * ch, do))


def lancir_expected(c, sl, new_dl):
    """Upstream CLancIR on the same padded source, into an identically pre-filled destination."""
    sw, sh, nw, nh, ti, to, kw = c
    kw = {k: v for k, v in kw.items() if k != "C"}
    ref = new_dl()
    r, _ = o.lancir_ref(sl.view(), nw, nh, to, srcssize=sl.pitch, newssize=ref.pitch, dst=ref.view(), **kw)
    assert r == nh
    return ref


needs_ref = pytest.mark.skipif(not o.have_ref(), reason="needs oracle/_ref (upstream CLancIR)")


@needs_ref
@pytest.mark.parametrize("layout", list(LANCIR_LAYOUTS))
@pytest.mark.parametrize("c", LANCIR_CASES, ids=_lancir_id)
def test_lancir_device_layouts(c, layout):
    sw, sh, nw, nh, ti, to, kw = c
    ch = kw.get("C", 4)
    sl, new_dl = lancir_layouts(c, layout)
    ref = lancir_expected(c, sl, new_dl)
    dl = new_dl()
    h = ab.host_lib().lancirb200_host_desc_create(o.T_OF[np.dtype(ti)], o.T_OF[np.dtype(to)], sw, sh, nw, nh, ch,
                                                  kw.get("kx", 0.0), kw.get("ky", 0.0), 0.0, 0.0, 3.0)
    assert h
    L, pl = lib(), C.c_void_p()
    try:
        _ok(L.lancirb200_plan_create(C.c_void_p(ab.host_lib().lancirb200_host_desc_get(h)), C.byref(pl)))
        b = C.c_size_t()
        _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(b)))
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(b.value)
        _ok(L.lancirb200_resize_device(pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None))
        import torch
        torch.cuda.synchronize()
        back = d_dst.cpu().numpy().view(dl.backing.dtype)
        assert tail_damage(ws, b.value) == 0
    finally:
        if pl.value:
            L.lancirb200_plan_destroy(pl)
        ab.host_lib().lancirb200_host_desc_free(h)
    # the whole destination buffer, guards and padding included, byte for byte
    assert np.array_equal(back.view(np.uint8), ref.backing.view(np.uint8))


@needs_ref
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("layout", ["vec-in-vec-out", "scalar-in-scalar-out"])
@pytest.mark.parametrize("c", LANCIR_CASES, ids=_lancir_id)
def test_lancir_host_scanline_sizes(c, layout, pinned):
    """CLancIR::resizeImage with SrcSSize / NewSSize on padded buffers = upstream, byte for byte."""
    sw, sh, nw, nh, ti, to, kw = c
    kw = dict(kw)
    kw.pop("C", None)
    sl, new_dl = lancir_layouts(c, layout, seed=10)
    ref = lancir_expected(c, sl, new_dl)
    dl = new_dl()
    if pinned:
        sl2, dl2 = cs.Layout(cs.host_array(sl.backing.size, sl.backing.dtype, True), sl.origin, sl.pitch, sl.shape), \
            cs.Layout(cs.host_array(dl.backing.size, dl.backing.dtype, True), dl.origin, dl.pitch, dl.shape)
        sl2.backing[:] = sl.backing
        dl2.backing[:] = dl.backing
        sl, dl = sl2, dl2
    r, _ = ab.CLancIR().resizeImage(sl.view(), nw, nh, ab.CLancIRParams(SrcSSize=sl.pitch, NewSSize=dl.pitch, **kw),
                                    out_dtype=to, NewBuf=dl.view())
    assert r == nh
    assert np.array_equal(dl.backing.view(np.uint8), ref.backing.view(np.uint8))


# ---- routing: each layout runs the kernel it is meant to cover ------------------------------------

KERNELS = ["stream_pass_kernel", "fast_pass_kernel", "generic_pass_kernel", "widen_channels_kernel",
           "narrow_channels_kernel", "lancir_col4_kernel", "lancir_col_kernel", "lancir_row4_kernel",
           "lancir_row_kernel"]


def launched_kernels(fn):
    """Names (from KERNELS) of the CUDA kernels fn() launched, in launch order; None when the
    profiler records no kernel activity on this machine."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = []
    for e in prof.events():
        for k in KERNELS:
            if re.search(r"\b%s\b" % k, e.name):
                evs.append((e.time_range.start, k))
                break
    if not evs:
        return None
    return [k for _, k in sorted(evs)]


S, F, G = "stream_pass_kernel", "fast_pass_kernel", "generic_pass_kernel"
W, N = "widen_channels_kernel", "narrow_channels_kernel"
ROUTES = [
    # (case, layout, kernel family, kernels launched in order)
    (CFG3_DIL, "L0-packed", 0, [S, S]),
    (CFG3_DIL, "L1-src-pad4", 0, [S, S]),
    (CFG3_DIL, "L2-src-pitch-not4", 0, [G, S]),
    (CFG3_DIL, "L3-src-offset1", 0, [G, S]),
    (CFG3_DIL, "L4-dst-pad2", 0, [S, S]),
    (CFG3_DIL, "L5-dst-odd", 0, [S, G]),
    (CFG3_DIL, "L5-dst-offset1", 0, [S, G]),
    (CFG3_DIL, "L6-src-offset1-dst-pad2", 0, [G, S]),
    (CFG3_DIL, "L6-src-pad4-dst-odd", 0, [S, G]),
    (CFG3_DIL, "L0-packed", 2, [F, F]),
    (CFG3_DIL, "L3-src-offset1", 2, [G, F]),
    (CFG3_DIL, "L5-dst-odd", 2, [F, G]),
    (CFG3_DIL, "L0-packed", 1, [G, G]),
    (TILE, "L0-packed", 0, [F, F]),
    (TILE, "L2-src-pitch-not4", 0, [G, F]),
    (TILE, "L6-src-pad4-dst-odd", 0, [F, G]),
    (RGB, "L0-packed", 2, [W, F, F, N]),
    (RGB, "L3-src-offset1", 2, [W, F, F, N]),  # widened copies are aligned whatever the caller's layout
    (RGB, "L0-packed", 1, [G, G]),
    (GRAY, "L0-packed", 1, [G, G]),
]


def route_failures():
    """(case, layout, kernels launched, kernels wanted) of each call that runs other kernels than it is meant to
    cover; None when the profiler records no kernel activity."""
    import torch
    failures = []
    for case, layout, family, want in ROUTES:
        sl, dl = make_layouts(case, layout)
        with avir_plan(case, family) as (L, pl):
            n = plan_workspace(L, pl)
            d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
            got = launched_kernels(lambda: _ok(L.avirb200_resize_device(
                pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None)))
        if got is None:
            return None
        if got != want:
            failures.append((cs.case_id(case), layout, family, got, want))
    for c in LANCIR_CASES[:1]:
        sw, sh, nw, nh, ti, to, kw = c
        for layout, (col, row) in {"vec-in-vec-out": ("lancir_col4_kernel", "lancir_row4_kernel"),
                                   "scalar-in-vec-out": ("lancir_col_kernel", "lancir_row4_kernel"),
                                   "vec-in-scalar-out": ("lancir_col4_kernel", "lancir_row_kernel"),
                                   "scalar-in-scalar-out": ("lancir_col_kernel", "lancir_row_kernel")}.items():
            sl, new_dl = lancir_layouts(c, layout)
            dl = new_dl()
            h = ab.host_lib().lancirb200_host_desc_create(o.T_OF[np.dtype(ti)], o.T_OF[np.dtype(to)], sw, sh, nw, nh,
                                                          4, 0.0, 0.0, 0.0, 0.0, 3.0)
            L, pl = lib(), C.c_void_p()
            try:
                _ok(L.lancirb200_plan_create(C.c_void_p(ab.host_lib().lancirb200_host_desc_get(h)), C.byref(pl)))
                b = C.c_size_t()
                _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(b)))
                d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(b.value)
                got = launched_kernels(lambda: _ok(L.lancirb200_resize_device(
                    pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None)))
            finally:
                if pl.value:
                    L.lancirb200_plan_destroy(pl)
                ab.host_lib().lancirb200_host_desc_free(h)
            if got != [col, row]:
                failures.append(("lancir", layout, got, [col, row]))
    torch.cuda.synchronize()
    return failures


def test_layouts_route_to_the_kernels_they_cover():
    """Run in a child process: a profiler session leaves state behind in the process that runs it, so that
    whether this one records kernels would depend on which tests ran before it."""
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_layouts as t; "
            "print(json.dumps(t.route_failures()))" % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    failures = json.loads(r.stdout.strip().splitlines()[-1])
    if failures is None:
        pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
    assert not failures, failures
