"""CLancIR with double and uint32_t buffers on the GPU (run with -m gpu on an H100).

Every comparison is against upstream CLancIR compiled in-tree (oracle/_ref/liblancir_types_ref.so), or the
oracle's C port (oracle/liblancir_types_port.so) where that is absent (test_lancir_types.py pins the port to upstream on these types), with 0 mismatching elements: NaN
positions must match, payloads need not (cases.value_mismatch).  The kernels read and write the new types
themselves, on the 4-channel vector kernels (pixel-aligned buffers) and the scalar kernels alike."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import cases as cs
import lancir_types_oracle as lo
from lancir_types_oracle import expected, lancir_plan
from test_gpu_lancir_window import full_device, window_in_place
from test_gpu_layouts import (LANCIR_LAYOUTS, _ok, _src_pitch, dptr, guarded_workspace, launched_kernels,
                              tail_damage, to_device)
from test_gpu_parity import LANCIR as PARITY_CASES
from test_gpu_window import upload
from test_lancir_types import NEW, NEW_PAIRS, TYPES, fixture_files, pid, type_image, value_source
from test_window import crop, window_set

pytestmark = pytest.mark.gpu

u8, u16, f32, f64, u32 = np.uint8, np.uint16, np.float32, np.float64, np.uint32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
mismatch = cs.value_mismatch


def front_end(src, nw, nh, to, kw=None):
    """avir::CLancIR::resizeImage through the host C API (the Python driver takes no double buffers)."""
    r, got = lo.front_end(src, nw, nh, to, kw)
    assert r == nh
    return got


def check_windows(src, nw, nh, to, kw, wins, ref):
    """The whole image on the device equals ref, every window (its source the footprint inside the resident
    whole image) the crop of the whole image."""
    sh, sw, ch = src.shape
    with lancir_plan(sw, sh, nw, nh, ch, src.dtype, to, kw) as (L, pl, _):
        d_src = upload(src)
        full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, to)
        assert mismatch(ref, full) == 0
        for win in wins:
            got = window_in_place(L, pl, d_src, sw, ch, src.dtype, to, win)
            assert mismatch(crop(full, win), got) == 0, win


# ---- against upstream: every new pair x the LANCIR parity geometries, and a seeded sweep ------------------------

@pytest.mark.parametrize("ti,to", NEW_PAIRS, ids=pid)
@pytest.mark.parametrize("sw,sh,nw,nh,kw", [c[:4] + (c[6],) for c in PARITY_CASES],
                         ids=lambda v: None if not isinstance(v, dict) else ("C%d" % v.get("C", 4)) + "".join(
                             "-%s%s" % kv for kv in sorted(v.items()) if kv[0] != "C"))
def test_new_pairs_bit_exact(sw, sh, nw, nh, kw, ti, to):
    kw = dict(kw)
    src = type_image(sh, sw, kw.pop("C", 4), ti, seed=3)
    assert mismatch(expected(src, nw, nh, to, kw), front_end(src, nw, nh, to, kw)) == 0


def test_sweep_all_types():
    """60 seeded calls: 1..4 channels, la 2 .. 5, both directions, offsets, explicit steps, all five types."""
    rng = np.random.default_rng(23)
    for it in range(60):
        ch = int(rng.integers(1, 5))
        sw, sh = int(rng.integers(2, 120)), int(rng.integers(2, 120))
        nw, nh = int(rng.integers(1, 200)), int(rng.integers(1, 200))
        ti, to = TYPES[int(rng.integers(0, 5))], TYPES[int(rng.integers(0, 5))]
        kw = {"la": float(rng.choice([2.0, 2.5, 3.0, 4.0, 5.0]))}
        if rng.random() < 0.3:
            kw["kx"], kw["ky"] = float(rng.choice([0.5, 0.8, 1.7, -1.3])), float(rng.choice([0.6, 1.0, 2.2, -0.9]))
        if rng.random() < 0.3:
            kw["ox"], kw["oy"] = float(rng.uniform(-1, 1)), float(rng.uniform(-1, 1))
        src = (value_source if ti in NEW and rng.random() < 0.3 else type_image)(sh, sw, ch, ti, 700 + it)
        got = front_end(src, nw, nh, to, kw)
        assert mismatch(expected(src, nw, nh, to, kw), got) == 0, (sw, sh, nw, nh, ch, pid(ti), pid(to), kw)


@pytest.mark.parametrize("f", fixture_files())
def test_fixtures(f):
    z = np.load(os.path.join(cs.GOLDEN, f))
    sw, sh, nw, nh = [int(v) for v in z["geom"]]
    assert mismatch(z["out"], front_end(z["src"], nw, nh, z["out"].dtype)) == 0


@pytest.mark.parametrize("ti,to", [(f64, f64), (u32, u32), (u8, f64)], ids=pid)
def test_full_size(ti, to):
    """8K -> 4K RGBA, device-resident (the vector kernels)."""
    import torch
    sw, sh, nw, nh, ch = 7680, 4320, 3840, 2160, 4
    src = type_image(sh, sw, ch, ti, seed=5)
    want = expected(src, nw, nh, to)
    with lancir_plan(sw, sh, nw, nh, ch, ti, to, {}) as (L, pl, _):
        got = full_device(L, pl, upload(src), sw, sh, nw, nh, ch, to)
    assert mismatch(want, got) == 0
    torch.cuda.empty_cache()


# ---- buffer layouts: the four LANCIR_LAYOUTS, guards, workspace tail, source untouched; the host form ----------

LAYOUT_CASES = [
    (96, 54, 48, 27, f64, f64, {}),
    (64, 48, 103, 77, u32, u32, {}),
    (64, 64, 16, 16, u8, f64, {}),
    (50, 30, 33, 17, f64, u32, {}),
    (77, 51, 47, 29, u32, f32, {"C": 3, "kx": 1.3, "ky": 2.2}),
    (96, 54, 48, 27, f64, u8, {"C": 1}),
]


def _lid(c):
    sw, sh, nw, nh, ti, to, kw = c
    return "%dx%d-%dx%d-%s-%s-c%d" % (sw, sh, nw, nh, pid(ti), pid(to), kw.get("C", 4))


def layouts(src, nw, nh, to, layout, pinned=False):
    sk, so, dmod, do = LANCIR_LAYOUTS[layout]
    sh, sw, ch = src.shape
    p = nw * ch + 4
    p += (dmod - p) % 4
    return (cs.source_layout(src, _src_pitch(sw * ch, sk) - sw * ch, so, pinned=pinned),
            cs.guarded_dest((nh, nw, ch), to, p - nw * ch, do, pinned=pinned))


@pytest.mark.parametrize("layout", list(LANCIR_LAYOUTS))
@pytest.mark.parametrize("c", LAYOUT_CASES, ids=_lid)
def test_device_layouts(c, layout):
    import torch
    sw, sh, nw, nh, ti, to, kw = c
    kw = dict(kw)
    ch = kw.pop("C", 4)
    src = type_image(sh, sw, ch, ti, seed=9)
    want = expected(src, nw, nh, to, kw)
    sl, dl = layouts(src, nw, nh, to, layout)
    with lancir_plan(sw, sh, nw, nh, ch, ti, to, kw) as (L, pl, _):
        n = C.c_size_t()
        _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
        d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n.value)
        _ok(L.lancirb200_resize_device(pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None))
        torch.cuda.synchronize()
        back = d_dst.cpu().numpy().view(dl.backing.dtype)
        assert mismatch(want, np.ascontiguousarray(dl.view(back))) == 0
        assert cs.guard_damage(dl, back) == 0, "destination guard bytes overwritten"
        assert tail_damage(ws, n.value) == 0, "store past lancirb200_plan_workspace_bytes"
        assert np.array_equal(d_src.cpu().numpy(), sl.backing.view(np.uint8)), "source buffer written"


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("layout", ["vec-in-vec-out", "scalar-in-scalar-out"])
@pytest.mark.parametrize("c", LAYOUT_CASES, ids=_lid)
def test_host_scanline_sizes(c, layout, pinned):
    sw, sh, nw, nh, ti, to, kw = c
    kw = dict(kw)
    ch = kw.pop("C", 4)
    src = type_image(sh, sw, ch, ti, seed=10)
    want = expected(src, nw, nh, to, kw)
    sl, dl = layouts(src, nw, nh, to, layout, pinned)
    r, _ = lo.front_end(sl.view(), nw, nh, to, kw, srcssize=sl.pitch, newssize=dl.pitch, dst=dl.view())
    assert r == nh
    assert mismatch(want, np.ascontiguousarray(dl.view())) == 0
    assert cs.guard_damage(dl) == 0
    assert mismatch(src, np.ascontiguousarray(sl.view())) == 0, "source buffer written"


def route_failures():
    """(pair, layout, kernels launched, kernels wanted) of each call that runs other kernels than it is meant
    to cover; None when the profiler records no kernel activity."""
    import torch
    sw, sh, nw, nh = 96, 54, 48, 27
    failures = []
    for ti, to in [(f64, f64), (u32, u32)]:
        src = type_image(sh, sw, 4, ti, seed=9)
        with lancir_plan(sw, sh, nw, nh, 4, ti, to, {}) as (L, pl, _):
            n = C.c_size_t()
            _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
            ws = torch.empty(n.value, dtype=torch.uint8, device="cuda")
            for off, want in [(0, ["lancir_col4_kernel", "lancir_row4_kernel"]),
                              (1, ["lancir_col_kernel", "lancir_row_kernel"])]:   # one element in: unaligned
                sl = cs.source_layout(src, 0, off)
                dl = cs.guarded_dest((nh, nw, 4), to, 0, off)
                d_src, d_dst = to_device(sl), to_device(dl)
                got = launched_kernels(lambda: _ok(L.lancirb200_resize_device(
                    pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch, ws.data_ptr(), None)))
                if got is None:
                    return None
                if got != want:
                    failures.append(("%s-%s" % (pid(ti), pid(to)), off, got, want))
    torch.cuda.synchronize()
    return failures


def test_route_to_the_kernels_they_cover():
    """Run in a child process: a profiler session leaves state behind in the process that runs it."""
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_lancir_types as t; "
            "print(json.dumps(t.route_failures()))" % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    failures = json.loads(r.stdout.strip().splitlines()[-1])
    if failures is None:
        pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
    assert not failures, failures


# ---- windows: every window equals the crop of the whole image, device and host forms --------------------------

WINDOW_CASES = [(96, 54, 48, 27, 4, {}), (64, 48, 103, 77, 3, {}), (77, 51, 47, 29, 1, {"la": 2.0}),
                (50, 30, 33, 17, 2, {"kx": 1.3, "ky": 2.2})]


@pytest.mark.parametrize("ti,to", NEW_PAIRS, ids=pid)
@pytest.mark.parametrize("g", WINDOW_CASES, ids=lambda g: "%dx%d-%dx%d-c%d" % g[:5])
def test_windows(g, ti, to):
    sw, sh, nw, nh, ch, kw = g
    src = type_image(sh, sw, ch, ti, seed=4)
    want = expected(src, nw, nh, to, kw)
    wins = window_set(nw, nh, seed=sw + ch)
    check_windows(src, nw, nh, to, kw, wins, ref=want)
    for win in wins[::2]:
        r, got = lo.front_end_window(src, nw, nh, to, win, kw)
        assert r == win[3] and mismatch(crop(want, win), got) == 0, win


# ---- the value domain, on the vector and the scalar kernels ----------------------------------------------------

@pytest.mark.parametrize("to", TYPES, ids=pid)
@pytest.mark.parametrize("ti", NEW, ids=pid)
def test_value_domain(ti, to):
    import torch
    for sw, sh, nw, nh, ch in [(70, 50, 33, 23, 4), (40, 30, 61, 47, 4), (70, 50, 33, 23, 3), (70, 50, 29, 19, 1)]:
        src = value_source(sh, sw, ch, ti, seed=ch + sw)
        want = expected(src, nw, nh, to)
        with lancir_plan(sw, sh, nw, nh, ch, ti, to, {}) as (L, pl, _):
            assert mismatch(want, full_device(L, pl, upload(src), sw, sh, nw, nh, ch, to)) == 0
            if ch == 4:   # one element in: the scalar kernels
                sl, dl = layouts(src, nw, nh, to, "scalar-in-scalar-out")
                n = C.c_size_t()
                _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
                d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n.value)
                _ok(L.lancirb200_resize_device(pl, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch,
                                               ws.data_ptr(), None))
                torch.cuda.synchronize()
                back = d_dst.cpu().numpy().view(dl.backing.dtype)
                assert mismatch(want, np.ascontiguousarray(dl.view(back))) == 0
                assert cs.guard_damage(dl, back) == 0


def test_nan_in_a_u32_row_tail():
    """A 3-channel uint32_t destination 33 pixels wide has a 3-element half-up tail per row.  Where NaN reaches
    an element, the tail holds x86's (int)NaN, 2147483648, and the body the clamp's 65535."""
    sw, sh, nw, nh, ch = 70, 40, 33, 20, 3
    src = type_image(sh, sw, ch, f64, seed=6)
    src[:, sw - 2] = np.nan        # a NaN column at the right edge
    src[sh // 2, 5, 1] = np.nan    # and one sample far from it
    got = front_end(src, nw, nh, u32)
    assert mismatch(expected(src, nw, nh, u32), got) == 0
    nan = np.isnan(front_end(src, nw, nh, f32)).reshape(nh, nw * ch)
    flat = got.reshape(nh, nw * ch)
    tail = np.zeros_like(nan)
    tail[:, (nw * ch) & ~3:] = True
    assert (nan & tail).any() and (nan & ~tail).any()
    assert (flat[nan & tail] == 2147483648).all()
    assert (flat[nan & ~tail] == 65535).all()


# ---- the C++ front-end program -----------------------------------------------------------------------------------

def test_types_program_writes_upstream_bits(tmp_path):
    from test_lancir_types import build_types_program
    exe = build_types_program()
    src_d = type_image(64, 96, 4, f64, seed=21)
    src_u = value_source(64, 96, 3, u32, seed=22)
    src_d.tofile(str(tmp_path / "in_f64.bin"))
    src_u.tofile(str(tmp_path / "in_u32.bin"))
    r = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    got = np.fromfile(str(tmp_path / "out_f64_f64.bin"), f64).reshape(32, 48, 4)
    assert mismatch(expected(src_d, 48, 32, f64), got) == 0
    got = np.fromfile(str(tmp_path / "out_u32_u32.bin"), u32).reshape(41, 61, 3)
    assert mismatch(expected(src_u, 61, 41, u32), got) == 0
    got = np.fromfile(str(tmp_path / "out_win.bin"), u32).reshape(11, 20, 4)
    assert mismatch(crop(expected(src_d, 48, 32, u32), (5, 3, 20, 11)), got) == 0
