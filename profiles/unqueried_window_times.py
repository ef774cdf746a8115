#!/usr/bin/env python
"""Device time of a destination window whose range was queried first (its passes on the tile kernel)
against the same window on a twin plan that never saw it queried (its passes on the generic kernel:
avirb200_resize_window_device builds no table inside a launch).  CUDA events, L2 flushed before every
call, 3 warm-ups, the two calls alternated, median of N.

    python profiles/unqueried_window_times.py [--n 30] [--win 1920 1080]

The chain is one the streaming kernel does not take (a non-integer ratio, 1.5 x 1.5), so that the
queried window runs on the tile kernel; both windows must give the same bytes.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402
import avir_b200 as ab  # noqa: E402

GEOM = (1, 7680, 4320, 5120, 2880, np.uint8, np.uint8, 8)  # fpclass, sw, sh, nw, nh, tin, tout, resbits


class WindowInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_x0", "src_w", "src_y0", "src_h", "mid_row0", "mid_rows")]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(n, ww, wh):
    fp, sw, sh, nw, nh, ti, to, rb = GEOM
    ch = 4
    lib = ab.lib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    lib.avirb200_plan_kernel_paths.argtypes = [vp]
    lib.avirb200_window_query.argtypes = [vp, i, i, i, i, vp]
    lib.avirb200_window_workspace_bytes.argtypes = [vp, i, i, i, i, vp]
    lib.avirb200_resize_window_device.argtypes = [vp, i, i, i, i, vp, sz, vp, sz, vp, vp]
    rs = ab.CImageResizer(rb, 0, 0, fp)
    h, dp, modes = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, ab.CImageResizerVars())
    queried, fresh = C.c_void_p(), C.c_void_p()
    for p in (queried, fresh):
        assert lib.avirb200_plan_create(C.c_void_p(dp), C.byref(p)) == 0, lib.avirb200_last_error()
    paths = lib.avirb200_plan_kernel_paths(queried)
    assert paths & 0xC == 0xC and paths & 0x3 == 0, paths  # both passes on the tile kernel, not streaming
    g = torch.Generator(device="cuda").manual_seed(1)
    d_src = torch.randint(0, 256, (sh, sw, ch), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    win = ((nw - ww) // 2 + 1, (nh - wh) // 2 + 1, ww, wh)  # centred, at odd offsets
    fi, wn = WindowInfo(), C.c_size_t()
    assert lib.avirb200_window_query(queried, *win, C.byref(fi)) == 0, lib.avirb200_last_error()
    assert lib.avirb200_window_workspace_bytes(queried, *win, C.byref(wn)) == 0
    outs = [torch.zeros((wh, ww, ch), device="cuda", dtype=torch.uint8) for _ in range(2)]
    wss = [torch.empty(wn.value, dtype=torch.uint8, device="cuda") for _ in range(2)]
    w_src = d_src.data_ptr() + (fi.src_y0 * sw + fi.src_x0) * ch
    st = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def call(k):
        pl = (queried, fresh)[k]
        assert lib.avirb200_resize_window_device(pl, *win, w_src, sw * ch, outs[k].data_ptr(), ww * ch,
                                                 wss[k].data_ptr(), st) == 0, lib.avirb200_last_error()

    def timed(k):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call(k)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(3):
        call(0)
        call(1)
    tq, tf = [], []
    for _ in range(n):  # alternated
        tq.append(timed(0))
        tf.append(timed(1))
    torch.cuda.synchronize()
    same = bool(torch.equal(outs[0], outs[1]))
    qms, fms = sorted(tq)[n // 2], sorted(tf)[n // 2]
    rec = {"geometry": "%dx%d->%dx%d RGBA u8, fpclass %d" % (sw, sh, nw, nh, fp), "window": list(win),
           "footprint": [fi.src_x0, fi.src_w, fi.src_y0, fi.src_h], "kernel_paths": paths, "same_bytes": same,
           "n": n, "queried_tile_ms": round(qms, 4), "unqueried_generic_ms": round(fms, 4),
           "generic_over_tile": round(fms / qms, 3),
           "queried_ms_spread": [round(min(tq), 4), round(max(tq), 4)],
           "unqueried_ms_spread": [round(min(tf), 4), round(max(tf), 4)], "build_modes": list(modes)}
    for p in (queried, fresh):
        lib.avirb200_plan_destroy(p)
    rs.free_descriptor(h)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--win", nargs=2, type=int, default=[1920, 1080])
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}))
    print(json.dumps(run(a.n, *a.win)))


if __name__ == "__main__":
    main()
