"""The value domain on the GPU (run with -m gpu on an H100): samples outside [0, 1], beyond int32 once
scaled to the output range, +-Inf, NaN, +-FLT_MAX, subnormals, +-0.0, rounding ties, every u8 and u16
code -- through every fpclass, output type, chain and kernel family.

The output stage is where x86 and the device differ: upstream's round() is x86's (int), which yields
INT_MIN for NaN and outside int32, where the device's conversions saturate.  The inputs come from
cases.value_image; the reference is upstream (oracle/_ref), or where it is absent the value_*.npz
fixtures upstream wrote.  Comparison (cases.value_mismatch): integers exactly, floats bit for bit
with any NaN matching any NaN -- upstream passes a NaN's payload through, the device's FADD / FMUL
return the canonical NaN -- so NaN positions, +-0 and +-Inf all count.

Non-finite samples spread (Inf times a negative lobe plus Inf is NaN), so they are sparse, on images
large enough that most outputs stay finite; a NaN where upstream has a number (a kernel skipping a
zero tap that upstream multiplies by Inf) shows up as a mismatch.
"""
import ctypes as C
import os

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
import test_gpu_layouts as gl

pytestmark = pytest.mark.gpu

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
needs_ref = pytest.mark.skipif(not o.have_ref(), reason="needs oracle/_ref (upstream); the fixtures still run")


@pytest.fixture(params=[0, 2, 1], ids=["product", "tile", "generic"])
def kernel_path(request):
    """Every pass of the host calls on the product's kernel choice, the tile kernel, the generic kernel."""
    ab.set_option(ab.OPT_KERNEL_FAMILY, request.param)
    yield request.param
    ab.set_option(ab.OPT_KERNEL_FAMILY, -1)


# streaming chains (explicit build modes: the automatic one depends on the image size)
CFG3_DIL = (2, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1})
CFG3_DIL_U8 = (0, 192, 108, 96, 54, 4, f32, u8, 8, {"buildmode": 1})
CFG3_F4 = (1, 192, 108, 96, 54, 4, f32, u8, 8, {"buildmode": 0})
CFG2 = (0, 96, 64, 192, 128, 4, f32, u8, 8, {"buildmode": 1})
CFG4 = (1, 256, 192, 64, 48, 4, f32, u16, 16, {"buildmode": 0})
CFG5 = (2, 256, 192, 64, 48, 4, f32, u8, 8, {"buildmode": 1})
TILE = (0, 150, 90, 100, 55, 4, f32, u8, 8, {"buildmode": 1})      # irregular ratio
UPSAMPLE = (0, 96, 64, 192, 128, 4, f32, u8, 8, {"buildmode": 0})  # filtered 2X upsample: generic kernel

FLOAT_CASES = [
    CFG3_DIL, CFG3_DIL_U8, CFG3_F4, CFG2, CFG4, CFG5, TILE, UPSAMPLE,
    (0, 192, 108, 96, 54, 4, f32, u16, 16, {"buildmode": 1}),
    (2, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1, "gamma": True}),       # lin2srgb_batch fallback
    (2, 192, 108, 96, 54, 4, f32, u8, 8, {"buildmode": 1, "gamma": True, "alpha": 3}),
    (1, 96, 64, 192, 128, 4, f32, u16, 16, {"buildmode": 1}),
    (0, 256, 192, 64, 48, 4, f32, u8, 8, {"buildmode": 0}),
    (2, 256, 192, 64, 48, 4, f32, f64, 16, {"buildmode": 1}),
    (2, 150, 90, 100, 55, 4, f32, f32, 16, {}),
    (2, 96, 64, 192, 128, 4, f32, f32, 16, {"buildmode": 0}),
    # 1-3 channels, widened onto the 4-channel kernels
    (0, 192, 144, 96, 72, 3, f32, u8, 8, {}),
    (1, 192, 108, 96, 54, 1, f32, f32, 16, {}),
    (0, 192, 108, 96, 54, 2, f32, u16, 16, {"gamma": True}),
    # bit-depth truncation (TrMul != 1), double output
    (0, 130, 100, 100, 75, 4, f32, u8, 6, {}),
    (2, 192, 108, 96, 54, 4, f32, u16, 12, {"buildmode": 1}),
    (0, 120, 80, 60, 40, 3, f32, f64, 16, {"gamma": True}),
    # error diffusion (fpclass 3..5): round() inside the recursion
    (3, 160, 120, 80, 60, 4, f32, u8, 8, {}),
    (4, 160, 120, 80, 60, 4, f32, u16, 16, {}),
    (5, 160, 120, 80, 60, 4, f32, u8, 6, {"gamma": True, "alpha": 3}),
    (3, 100, 60, 150, 77, 3, f32, u8, 6, {}),
]
# float64 sources: 1e39 / 1e300 (Inf once cast to float) and double subnormals on top of the kind
DOUBLE_CASES = [
    (1, 192, 108, 96, 54, 4, f64, f64, 16, {}),
    (2, 150, 90, 100, 55, 2, f64, u8, 8, {}),
    (0, 120, 80, 60, 40, 4, f64, u16, 16, {"gamma": True, "alpha": 3}),
]
# integer sources: every code (the u8 sRGB table, the double-precision u16 linearisation), all 0, all max
INT_CASES = [
    (2, 128, 128, 32, 32, 4, u8, u8, 8, {"gamma": True, "alpha": 3, "buildmode": 1}),
    (1, 128, 128, 64, 64, 4, u8, u8, 8, {"buildmode": 1}),
    (0, 128, 96, 64, 48, 3, u8, f32, 8, {"gamma": True}),
    (1, 256, 256, 64, 64, 4, u16, u16, 16, {"buildmode": 0}),
    (0, 256, 256, 128, 128, 4, u16, f32, 16, {"gamma": True, "alpha": 3}),
    (5, 256, 256, 128, 128, 2, u16, u8, 8, {"gamma": True}),
    (3, 128, 128, 64, 64, 4, u8, u8, 8, {}),
]
PAIRS = ([(c, k) for c in FLOAT_CASES for k in cs.VALUE_KINDS]
         + [(c, k) for c in DOUBLE_CASES for k in ("range", "nonfinite", "tiny")]
         + [(c, k) for c in INT_CASES for k in cs.INT_KINDS])

_want = {}


def expected(case, kind, src):
    """Upstream's output (computed once, shared by the three kernel families)."""
    key = (cs.case_id(case), kind)
    if key not in _want:
        _want[key] = cs.ref_output(case, src)
    return _want[key]


@needs_ref
@pytest.mark.parametrize("case,kind", PAIRS, ids=["%s-%s" % (cs.case_id(c), k) for c, k in PAIRS])
def test_value_domain_matches_upstream(case, kind, kernel_path):
    src = cs.value_image(case, kind)
    got = cs.gpu_output(case, src)
    assert cs.value_mismatch(expected(case, kind, src), got) == 0


def test_value_fixtures(kernel_path):
    """The value_*.npz fixtures (upstream's outputs, tests/golden/make_golden.py) on the GPU."""
    files = sorted(f for f in os.listdir(cs.GOLDEN) if f.startswith("value_") and f.endswith(".npz"))
    assert len(files) >= 6
    for f in files:
        z = np.load(os.path.join(cs.GOLDEN, f), allow_pickle=True)
        case = tuple(z["case"].tolist())
        case = case[:6] + (np.dtype(case[6]).type, np.dtype(case[7]).type) + case[8:]
        assert cs.value_mismatch(z["out"], cs.gpu_output(case, z["src"])) == 0, f


# ---- banded host call and the sharded schedule: halo rows carrying Inf and NaN ----------------------

BAND_CASES = [
    (0, 256, 216, 128, 108, 4, f32, u8, 8, {"buildmode": 1}),
    (2, 256, 216, 128, 108, 4, f32, f32, 16, {"buildmode": 1}),
]


def huge_and_nonfinite(case):
    """The "huge" image with the "nonfinite" kind's specials on top."""
    src = cs.value_image(case, "huge")
    nf = cs.value_image(case, "nonfinite", seed=12)
    sp = ~np.isfinite(nf) | (np.abs(nf) >= 3e38)
    src[sp] = nf[sp]
    return src


@needs_ref
@pytest.mark.parametrize("case", BAND_CASES, ids=cs.case_id)
def test_banded_host_call(case, kernel_path):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = huge_and_nonfinite(case)
    want = cs.ref_output(case, src)
    ab.set_option(ab.OPT_HOST_BANDS, 3)
    try:
        got = cs.gpu_output(case, src)
    finally:
        ab.set_option(ab.OPT_HOST_BANDS, -1)
    assert cs.value_mismatch(want, got) == 0


@needs_ref
@pytest.mark.parametrize("family", [0, 2, 1], ids=["product", "tile", "generic"])
@pytest.mark.parametrize("overlap", [3, 1])
@pytest.mark.parametrize("case", BAND_CASES, ids=cs.case_id)
def test_sharded_local(case, overlap, family):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = huge_and_nonfinite(case)
    want = cs.ref_output(case, src)
    sl, dl = cs.source_layout(src), cs.guarded_dest((nh, nw, ch), to)
    import torch
    with gl.avir_plan(case, family, {ab.OPT_OVERLAP_HALO: overlap}) as (L, pl):
        n = 0
        for r in range(3):
            b = C.c_size_t()
            gl._ok(L.avirb200_shard_workspace_bytes(pl, r, 3, C.byref(b)))
            n += b.value
        d_src, d_dst, ws = gl.to_device(sl), gl.to_device(dl), gl.guarded_workspace(n)
        gl._ok(L.avirb200_resize_sharded_local(pl, 3, gl.dptr(d_src, sl), sl.pitch, gl.dptr(d_dst, dl), dl.pitch,
                                               ws.data_ptr(), None))
        torch.cuda.synchronize()
        back = d_dst.cpu().numpy().view(dl.backing.dtype)
    assert cs.value_mismatch(want, np.ascontiguousarray(dl.view(back))) == 0
    assert cs.guard_damage(dl, back) == 0


# ---- LANCIR: clamps before it converts; the (W*C) & 3 tail rounds with (int)(v + 0.5f) --------------

LANCIR_CASES = [
    (96, 64, 48, 32, 4, u8), (96, 64, 48, 32, 4, u16), (96, 64, 48, 32, 4, f32),  # vector kernels
    (64, 48, 103, 77, 4, u8),
    (77, 51, 47, 29, 3, u8), (77, 51, 47, 29, 1, u16), (77, 51, 47, 29, 2, f32),  # (W*C) & 3 != 0
    (77, 51, 47, 29, 1, u8),
]


@needs_ref
@pytest.mark.parametrize("kind", ("range", "huge", "nonfinite", "tiny"))
@pytest.mark.parametrize("c", LANCIR_CASES, ids=lambda c: "%dx%d-%dx%d-c%d-%s" % (c[:5] + (np.dtype(c[5]).name,)))
def test_lancir_value_domain(c, kind):
    sw, sh, nw, nh, ch, to = c
    src = cs.value_image((0, sw, sh, nw, nh, ch, f32, to, 8, {}), kind)
    r, want = o.lancir_ref(src, nw, nh, to)
    assert r == nh
    r2, got = ab.CLancIR().resizeImage(src, nw, nh, out_dtype=to)
    assert r2 == nh
    assert cs.value_mismatch(want, got) == 0


# ---- routing: the product-order cases run the kernels they stand for -------------------------------

S, F, G = "stream_pass_kernel", "fast_pass_kernel", "generic_pass_kernel"
ROUTES = [(CFG3_DIL, [S, S]), (CFG3_DIL_U8, [S, S]), (CFG3_F4, [S, S]), (CFG4, [S, S]), (CFG5, [S, S]),
          (CFG2, [S, F]), (TILE, [F, F]), (UPSAMPLE, [G, G])]


def test_value_cases_route_to_their_kernels():
    failures = []
    for case, want in ROUTES:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        src = cs.value_image(case, "nonfinite")
        with gl.avir_plan(case) as (L, pl):
            sl, dl = cs.source_layout(src), cs.guarded_dest((nh, nw, ch), to)
            n = gl.plan_workspace(L, pl)
            d_src, d_dst, ws = gl.to_device(sl), gl.to_device(dl), gl.guarded_workspace(n)
            got = gl.launched_kernels(lambda: gl._ok(L.avirb200_resize_device(
                pl, gl.dptr(d_src, sl), sl.pitch, gl.dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None)))
        if got is None:
            pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
        if got != want:
            failures.append((cs.case_id(case), got, want))
    assert not failures, failures
