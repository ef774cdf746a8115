"""The contract every host entry point shares (run with -m gpu on an H100).

All six calls that take host buffers -- avirb200_resize_host, _window_host and _sharded_host, and CLancIR's
three -- stage through one path (avir_b200/csrc/host_call.cu): the same locks, device, stream, staging
buffers and copies.  Here:

* avirb200_resize_sharded_host of one rank, with padded pitches in pageable and page-locked memory, gives
  the bits of avirb200_resize_device on the whole image, for float, double and error-diffused plans;
* a pitch one element shorter than a row, source or destination, is AVIRB200_ERR_BAD_ARG on every host
  entry point, and the destination is left untouched (AVIR's resize_host unbanded and in 2 row bands
  through the pageable bounce buffers)."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
from test_gpu_layouts import CFG3_DIL, ERRD, F64, SHARD_CASES, _dst_pitch, _ok, _src_pitch, avir_plan
from test_gpu_lancir_window import lancir_plan
from test_gpu_window import full_device, upload, wlib

pytestmark = pytest.mark.gpu

u8 = np.uint8
ERR_BAD_ARG = -1


def hlib():
    L = wlib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    L.avirb200_resize_sharded_host.argtypes = [vp, vp, i, i, vp, sz, vp, sz]
    L.lancirb200_resize_host.argtypes = [vp, vp, sz, vp, sz]
    L.lancirb200_resize_window_host.argtypes = [vp, i, i, i, i, vp, sz, vp, sz]
    L.lancirb200_resize_sharded_host.argtypes = [vp, vp, i, i, vp, sz, vp, sz]
    return L


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


# ---- avirb200_resize_sharded_host, one rank ----------------------------------------------------------------

@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("case", [CFG3_DIL, F64, ERRD], ids=cs.case_id)
def test_sharded_host_one_rank_equals_resize_device(case, pinned):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case, seed=12)
    sl = cs.source_layout(src, _src_pitch(sw * ch, "padodd") - sw * ch, pinned=pinned)
    dl = cs.guarded_dest((nh, nw, ch), to, _dst_pitch(nw * ch, "odd") - nw * ch, pinned=pinned)
    with avir_plan(case) as (_, pl):
        L = hlib()
        want = full_device(L, pl, case, upload(src))
        _ok(L.avirb200_resize_sharded_host(pl, None, 0, 1, sl.view().ctypes.data, sl.pitch, dl.view().ctypes.data,
                                           dl.pitch))
    assert same_bits(want, dl.view())
    assert cs.guard_damage(dl) == 0


# ---- a pitch one element short, on every host entry point ---------------------------------------------------

AVIR_CASE = SHARD_CASES[0]  # 192 x 216 -> 96 x 108 RGBA float: two row bands of it are valid
LANCIR_GEOM = (96, 54, 48, 27, 4, u8, u8, {})
WIN = (5, 3, 40, 20)  # (x0, y0, w, h)
HOST_ENTRIES = ["avir-host", "avir-host-2-bands", "avir-window-host", "avir-sharded-host", "lancir-host",
                "lancir-window-host", "lancir-sharded-host"]


def _call(L, pl, entry, src, sp, dst, dp):
    x0, y0, w, h = WIN
    if entry.startswith("avir-host"):
        return L.avirb200_resize_host(pl, src, sp, dst, dp)
    return {"avir-window-host": lambda: L.avirb200_resize_window_host(pl, x0, y0, w, h, src, sp, dst, dp),
            "avir-sharded-host": lambda: L.avirb200_resize_sharded_host(pl, None, 0, 1, src, sp, dst, dp),
            "lancir-host": lambda: L.lancirb200_resize_host(pl, src, sp, dst, dp),
            "lancir-window-host": lambda: L.lancirb200_resize_window_host(pl, x0, y0, w, h, src, sp, dst, dp),
            "lancir-sharded-host": lambda: L.lancirb200_resize_sharded_host(pl, None, 0, 1, src, sp, dst, dp)}[entry]()


@pytest.mark.parametrize("short", ["src", "dst"])
@pytest.mark.parametrize("entry", HOST_ENTRIES)
def test_short_pitch_is_refused(entry, short):
    if entry.startswith("avir"):
        fp, sw, sh, nw, nh, ch, ti, to = AVIR_CASE[:8]
        plan = avir_plan(AVIR_CASE, 0, {ab.OPT_HOST_BANDS: 2 if entry == "avir-host-2-bands" else 1})
    else:
        sw, sh, nw, nh, ch, ti, to, kw = LANCIR_GEOM
        plan = lancir_plan(sw, sh, nw, nh, ch, ti, to, kw)
    dst_w = WIN[2] if entry.endswith("window-host") else nw
    # pageable buffers, large enough for the call at its correct pitches
    src = cs.make_input((0, sw, sh, nw, nh, ch, ti, to, 8, {}), seed=13)
    dst = np.full(nh * nw * ch * np.dtype(to).itemsize, cs.SENTINEL, u8)
    sp, dp = sw * ch, dst_w * ch
    if short == "src":
        sp -= 1
    else:
        dp -= 1
    with plan as handles:
        L, pl = hlib(), handles[1]
        rc = _call(L, pl, entry, src.ctypes.data, sp, dst.ctypes.data, dp)
        msg = L.avirb200_last_error().decode()
    assert rc == ERR_BAD_ARG, (rc, msg)
    assert "pitch" in msg, msg
    assert (dst == cs.SENTINEL).all(), "destination written"
