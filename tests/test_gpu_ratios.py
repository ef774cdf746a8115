"""Large downscale ratios, tiny destinations and extreme upscales on the GPU (run with -m gpu on an
H100), on every kernel family, against upstream (oracle/_ref; the C port where it is absent).

For downscaling, the planner puts a decimating FIR of about 7.5 R taps (R ~ k / 2) first, so the
source span one output reaches grows as about 19 k.  Both the tile and the generic kernel stage that
span per tile in shared memory: these cases cross each family's limit.  Past it the tile kernel
declines the pass, the generic kernel narrows its tile to one output and then to fewer lines, and a
plan that fits no family is refused at plan creation (include/avirb200.h, avirb200_plan_create).

One axis is made extreme on a strip source ((k n) x 24 -> n x 24, or the transpose) so that the
oracle stays cheap; the realistic thumbnails make both axes large.  0 mismatching elements
everywhere: integers exactly, floats bit for bit (cases.value_mismatch).
"""
import ctypes as C
import os

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_gpu_layouts import (avir_plan, check, dptr, guarded_workspace, launched_kernels, lib, make_layouts,
                              plan_workspace, tail_damage, to_device)

pytestmark = pytest.mark.gpu

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
ERR_UNSUPPORTED = -4


def _threads():
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 8
    return max(1, min(n, 16))


@pytest.fixture(params=[0, 2, 1], ids=["product", "tile", "generic"])
def kernel_path(request):
    """The product's kernel order, the tile kernel where it applies, and the generic kernel only."""
    ab.set_option(ab.OPT_KERNEL_FAMILY, request.param)
    yield request.param
    ab.set_option(ab.OPT_KERNEL_FAMILY, -1)


_expected = {}


def expected(case, seed=7, src=None):
    """Upstream's result for the case's seeded input (cached across kernel families)."""
    key = (cs.case_id(case), seed)
    if key not in _expected:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        if src is None:
            src = cs.make_input(case, seed=seed)
        if o.have_ref():
            want = o.ref_resize(src, nw, nh, to, fpclass=fp, resbits=rb, nthreads=_threads(), **cs.ref_kwargs(kw))
        else:
            want = cs.port_output(case, src)[0]
        _expected[key] = want
    return _expected[key]


def check_case(case, seed=7):
    src = cs.make_input(case, seed=seed)
    want = expected(case, seed, src)
    got = cs.gpu_output(case, src)
    assert cs.value_mismatch(want, got) == 0


# ---- the ratio ladder: one extreme axis on a strip -------------------------------------------------

LADDER_K = [16, 17, 20, 22, 24, 25, 28, 32, 48, 64, 100, 128, 200, 256]
STRIP_N = 24  # destination pixels along the extreme axis: a span of ~19 k is not clipped to the line


def strip(ratio, axis, ch, ti, fp=None, n=STRIP_N, rb=None, **kw):
    """(ratio n) x 24 -> n x 24 (axis "row") or its transpose (axis "col")."""
    if fp is None:
        fp = 2 if ti == f32 else 1
    if rb is None:
        rb = 16 if ti != u8 else 8
    if axis == "row":
        return (fp, ratio * n, 24, n, 24, ch, ti, ti, rb, kw)
    return (fp, 24, ratio * n, 24, n, ch, ti, ti, rb, kw)


LADDER = [strip(k, ax, ch, ti) for k in LADDER_K for ax in ("row", "col") for ch in (1, 2, 3, 4)
          for ti in (u8, f32)]


@pytest.mark.parametrize("case", LADDER, ids=cs.case_id)
def test_ratio_ladder(case, kernel_path):
    check_case(case)


# ---- realistic thumbnails: both axes large ----------------------------------------------------------

THUMBS = [
    (1, 4000, 3000, 125, 94, 4, u8, u8, 8, {}),
    (1, 3000, 4000, 94, 125, 4, u8, u8, 8, {}),
    (1, 4000, 3000, 125, 94, 3, u8, u8, 8, {}),
    (1, 3000, 4000, 94, 125, 3, u8, u8, 8, {}),
    (2, 7680, 4320, 256, 144, 4, f32, f32, 16, {}),
    (1, 4032, 3024, 126, 95, 4, u16, u16, 12, {}),
]


@pytest.mark.parametrize("case", THUMBS, ids=cs.case_id)
def test_thumbnails(case, kernel_path):
    check_case(case, seed=13)


# ---- tiny destinations, and the one beyond the documented bound ---------------------------------------

TINY = [
    (1, 4096, 16, 1, 16, 4, u8, u8, 8, {}),
    (1, 16, 4096, 16, 1, 4, u8, u8, 8, {}),
    (2, 2048, 2048, 1, 1, 4, f32, f32, 16, {}),
    (1, 8192, 8, 3, 8, 4, u8, u8, 8, {}),
    (1, 8192, 8, 3, 8, 1, u8, u8, 8, {}),
    (1, 11264, 4, 1, 4, 4, u8, u8, 8, {}),   # 4-channel line just inside the bound
    (1, 16384, 4, 1, 4, 3, u8, u8, 8, {}),   # 1..3 channels: the same line fits
    (1, 4, 16384, 4, 1, 2, u8, u8, 8, {}),
]


@pytest.mark.parametrize("case", TINY, ids=cs.case_id)
def test_tiny_destinations(case, kernel_path):
    check_case(case, seed=17)


REFUSED = [
    (1, 16384, 4, 1, 4, 4, u8, u8, 8, {}, "row pass"),
    (1, 4, 16384, 4, 1, 4, u16, u16, 16, {}, "column pass"),
]


@pytest.mark.parametrize("case", REFUSED, ids=lambda c: cs.case_id(c[:10]))
def test_beyond_the_bound_is_refused_at_plan_creation(case):
    """A 4-channel line of 16384 px to one pixel fits no kernel family: avirb200_plan_create says so
    (AVIRB200_ERR_UNSUPPORTED, naming the pass) and no kernel runs."""
    *c, what = case
    c = tuple(c)
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = c
    rs, v = cs.resizer_and_vars(c)
    h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, v)
    L, pl = lib(), C.c_void_p()
    try:
        assert L.avirb200_plan_create(C.c_void_p(dp), C.byref(pl)) == ERR_UNSUPPORTED
        assert not pl.value
        assert what in L.avirb200_last_error().decode()
    finally:
        if pl.value:
            L.avirb200_plan_destroy(pl)
        rs.free_descriptor(h)
    src = cs.make_input(c)
    got = launched_kernels(lambda: pytest.raises(ab.AvirB200Error, cs.gpu_output, c, src))
    if got is not None:
        assert got == []
    with pytest.raises(ab.AvirB200Error, match=what):
        cs.gpu_output(c, src)


# ---- the call surface at a large ratio ----------------------------------------------------------------

def _surface(k):
    n = 8
    return [
        # every class, error diffusion included
        strip(k, "row", 4, u8, fp=0, n=n), strip(k, "col", 4, u8, fp=1, n=n), strip(k, "row", 3, u8, fp=2, n=n),
        strip(k, "col", 4, u8, fp=3, n=n), strip(k, "row", 4, u8, fp=4, n=n), strip(k, "col", 2, u8, fp=5, n=n),
        # element types
        strip(k, "row", 4, u16, fp=1, n=n), strip(k, "col", 4, f32, fp=1, n=n),
        strip(k, "row", 3, f64, fp=1, n=n),
        # sRGB gamma, alpha first and last; a float source with input gamma (generic by design)
        strip(k, "row", 4, u8, fp=1, n=n, gamma=True, alpha=0), strip(k, "col", 4, u8, fp=2, n=n, gamma=True, alpha=3),
        strip(k, "row", 4, f32, fp=1, n=n, gamma=True), strip(k, "col", 3, f32, fp=2, n=n, gamma=True),
        # truncated bit depth, explicit negative k, offsets
        strip(k, "row", 4, u8, fp=1, n=n, rb=6), strip(k, "col", 4, u16, fp=0, n=n, rb=12),
        strip(k, "row", 4, f32, fp=2, n=n, k=-float(k)), strip(k, "col", 4, u8, fp=1, n=n, ox=0.37, oy=-0.21),
    ] + [strip(k, ("row", "col")[p % 2], 4, u8, fp=p % 3, n=n, params=p) for p in range(6)]


SURFACE = _surface(32) + _surface(100)


@pytest.mark.parametrize("case", SURFACE, ids=cs.case_id)
def test_call_surface_at_large_ratio(case, kernel_path):
    check_case(case, seed=19)


# ---- extreme upscales ---------------------------------------------------------------------------------

UPSCALES = [
    (1, 1, 1, 4096, 3, 4, u8, u8, 8, {}),
    (1, 7, 5, 3840, 2160, 4, u8, u8, 8, {}),
    (2, 2, 2000, 2000, 2000, 1, f32, f32, 16, {}),
    (1, 50, 40, 400, 300, 3, u8, u8, 8, {"buildmode": 0}),   # filtered upsample, k = 0.125
]


@pytest.mark.parametrize("case", UPSCALES, ids=cs.case_id)
def test_extreme_upscales(case, kernel_path):
    check_case(case, seed=23)


# ---- entry points on a large-ratio plan -----------------------------------------------------------------

TALL = strip(32, "col", 4, u8, n=96)           # 24 x 3072 -> 24 x 96: wide halos
TALL3 = strip(48, "col", 3, u16, n=64)
WIDE = strip(64, "row", 4, f32, n=32)


@pytest.mark.parametrize("bands", [2, 3, 7])
@pytest.mark.parametrize("case", [TALL, TALL3], ids=cs.case_id)
def test_banded_host_call_at_large_ratio(case, bands, kernel_path):
    src = cs.make_input(case, seed=29)
    ab.set_option(ab.OPT_HOST_BANDS, bands)
    try:
        got = cs.gpu_output(case, src)
    finally:
        ab.set_option(ab.OPT_HOST_BANDS, -1)
    assert cs.value_mismatch(expected(case, 29, src), got) == 0


FAMILIES = pytest.mark.parametrize("family", [0, 2, 1], ids=["product", "tile", "generic"])


@FAMILIES
@pytest.mark.parametrize("nranks", [2, 3])
@pytest.mark.parametrize("case", [TALL, TALL3], ids=cs.case_id)
def test_sharded_local_at_large_ratio(case, nranks, family):
    sl, dl = make_layouts(case, "L0-packed", seed=31)
    want = expected(case, ("sharded", 31), np.ascontiguousarray(sl.view()))
    with avir_plan(case, family) as (L, pl):
        n = 0
        for r in range(nranks):
            b = C.c_size_t()
            assert L.avirb200_shard_workspace_bytes(pl, r, nranks, C.byref(b)) == 0
            n += b.value
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
        assert L.avirb200_resize_sharded_local(pl, nranks, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch,
                                               ws.data_ptr(), None) == 0, L.avirb200_last_error().decode()
        check(want, dl, d_dst)
        assert tail_damage(ws, n) == 0


@FAMILIES
@pytest.mark.parametrize("layout", ["L0-packed", "L2-src-pitch-not4", "L6-src-pad4-dst-odd"])
@pytest.mark.parametrize("case", [WIDE, TALL, TALL3], ids=cs.case_id)
def test_split_passes_and_layouts_at_large_ratio(case, layout, family):
    """avirb200_resize_device and the row pass then the column pass, on padded and offset buffers
    with guarded destinations."""
    sl, dl = make_layouts(case, layout, seed=37)
    want = expected(case, ("layout", layout), np.ascontiguousarray(sl.view()))
    with avir_plan(case, family) as (L, pl):
        n = plan_workspace(L, pl)
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
        assert L.avirb200_resize_device(pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch,
                                        ws.data_ptr(), None) == 0, L.avirb200_last_error().decode()
        check(want, dl, d_dst, "resize_device")
        d_dst = to_device(dl)
        assert L.avirb200_row_pass_device(pl, dptr(d_src, sl), sl.pitch, ws.data_ptr(), None) == 0
        assert L.avirb200_col_pass_device(pl, ws.data_ptr(), dptr(d_dst, dl), dl.pitch, None) == 0
        check(want, dl, d_dst, "row pass + column pass")
        assert tail_damage(ws, n) == 0


@FAMILIES
@pytest.mark.parametrize("case", [WIDE, TALL3], ids=cs.case_id)
def test_batch_at_large_ratio(case, family):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    nf = 3
    sls = [cs.source_layout(cs.make_input(case, seed=40 + i), 0, i) for i in range(nf)]
    dls = [cs.guarded_dest((nh, nw, ch), to, 0, i % 2) for i in range(nf)]
    with avir_plan(case, family) as (L, pl):
        nb = plan_workspace(L, pl)
        d_srcs, d_dsts, ws = [to_device(s) for s in sls], [to_device(d) for d in dls], guarded_workspace(nb)
        sp = (C.c_void_p * nf)(*[dptr(t, s) for t, s in zip(d_srcs, sls)])
        dp = (C.c_void_p * nf)(*[dptr(t, d) for t, d in zip(d_dsts, dls)])
        assert L.avirb200_resize_device_batch(pl, nf, sp, sw * ch, dp, nw * ch, ws.data_ptr(), None) == 0
        for i in range(nf):
            check(expected(case, 40 + i, np.ascontiguousarray(sls[i].view())), dls[i], d_dsts[i], "frame %d" % i)
        assert tail_damage(ws, nb) == 0


WINDOWS = [
    (WIDE, (0, 0, 32, 24)),                          # the whole destination
    (WIDE, (5, 3, 20, 17)),
    (TALL, (2, 40, 19, 50)),
    (TINY[0], (0, 0, 1, 16)),                        # a window of a one-pixel-wide destination
    (TINY[0], (0, 5, 1, 7)),
    (TINY[1], (3, 0, 9, 1)),
]


@pytest.mark.parametrize("cw", WINDOWS, ids=lambda cw: "%s-w%d-%d-%d-%d" % ((cs.case_id(cw[0]),) + cw[1]))
def test_windows_at_large_ratio(cw, kernel_path):
    case, (x0, y0, w, h) = cw
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case, seed=43)
    want = expected(case, 43, src)
    rs, v = cs.resizer_and_vars(case)
    got = rs.resizeImageWindow(src, nw, nh, (x0, y0, w, h), kw.get("k", 0.0), v, out_dtype=to)
    assert cs.value_mismatch(np.ascontiguousarray(want[y0:y0 + h, x0:x0 + w]), got) == 0


# ---- which kernel runs ---------------------------------------------------------------------------------

F, G = "fast_pass_kernel", "generic_pass_kernel"
W, N = "widen_channels_kernel", "narrow_channels_kernel"
ROUTES = [
    # (case, the extreme axis's pass on the tile kernel, 1..3 channels widened onto the 4-channel kernels)
    (strip(16, "row", 4, u8, n=4), True, False),      # a 64-px line: the tile fits
    (strip(16, "col", 4, u16, n=4), True, False),
    (strip(100, "row", 4, u8), False, False),         # 2400 px to 24: it does not
    (strip(100, "col", 4, f32), False, False),
    ((1, 64, 64, 4, 4, 3, u8, u8, 8, {}), True, True),  # widened: the tiles of both passes fit
    (strip(100, "row", 3, u8), False, False),         # not widened: the image's own channels, generic
    (strip(100, "col", 1, f32), False, False),
]


def test_large_ratios_route_to_the_kernels_that_fit():
    """avirb200_plan_kernel_paths and the kernels resize_device launches (torch.profiler): a tile that
    fits keeps the tile kernel, one that does not runs the generic kernel, and a 1..3-channel plan
    whose tile does not fit keeps its own channel count."""
    import torch
    failures = []
    for case, tile, widened in ROUTES:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        row = sw > nw
        sl, dl = make_layouts(case, "L0-packed")
        with avir_plan(case) as (L, pl):
            paths = L.avirb200_plan_kernel_paths(pl)
            n = plan_workspace(L, pl)
            d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
            got = launched_kernels(lambda: L.avirb200_resize_device(
                pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None))
            check(expected(case, ("route",), np.ascontiguousarray(sl.view())), dl, d_dst)
        got_tile = bool(paths & (4 if row else 8))
        if got is not None:
            passes = [k for k in got if k not in (W, N)]
            assert len(passes) == 2, got
            ran = passes[0 if row else 1]
            got_widened = W in got
        else:
            ran, got_widened = (F if tile else G), widened
        if ch < 4 and not widened:
            assert n < nw * sh * 4 * 4, cs.case_id(case)   # the intermediate has the image's channel count
        if (got_tile, ran, got_widened) != (tile, F if tile else G, widened):
            failures.append((cs.case_id(case), paths, got, tile, widened))
    torch.cuda.synchronize()
    assert not failures, failures


# ---- CLancIR at large ratios: kernel lengths above 24 take the general loop --------------------------------

LANCIR = [(k, la, ch, ti) for k in (16, 32, 64, 128) for la in (2, 3, 5) for ch in (1, 4) for ti in (u8, f32)] + \
    [(24, 4, 2, u16), (100, 2, 3, u8), (48, 5, 3, f32)]


@pytest.mark.skipif(not o.have_ref(), reason="needs oracle/_ref (upstream CLancIR)")
@pytest.mark.parametrize("axis", ["row", "col"])
@pytest.mark.parametrize("c", LANCIR, ids=lambda c: "k%d-la%d-c%d-%s" % (c[0], c[1], c[2], np.dtype(c[3]).name))
def test_lancir_large_ratios(c, axis):
    k, la, ch, ti = c
    n = 12
    sw, sh, nw, nh = (k * n, 20, n, 20) if axis == "row" else (20, k * n, 20, n)
    src = o.lcg_image(sh, sw, ch, ti, seed=47)
    r, want = o.lancir_ref(src, nw, nh, ti, la=float(la))
    assert r == nh
    r2, got = ab.CLancIR().resizeImage(src, nw, nh, ab.CLancIRParams(la=float(la)))
    assert r2 == nh
    assert cs.value_mismatch(want, got) == 0
