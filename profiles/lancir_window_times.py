#!/usr/bin/env python
"""Device-resident time of a CLancIR destination window against the whole image (CUDA events, L2 flushed
before every call, 3 warm-ups, calls of the two alternated, median of N), with the window's algorithmic
bytes and their rate as a share of the H100 SXM's 3.35 TB/s data-sheet HBM3 bandwidth.

    python profiles/lancir_window_times.py [--n 30] [--win 1920 1080]

Setup: 8K -> 4K RGBA u8 (k = 2, 12 taps per axis).  Bytes of a call = source it reads + intermediate
written and read back + destination written: the whole image's src + 2 x mid (dst_h x src_w pixels of
floats) + dst, the window's footprint src + 2 x window mid (h x footprint-width pixels) + window dst (the
footprint from lancirb200_window_query).  The window is centred at odd offsets; its source is the
footprint inside the resident whole image (pitched rows: a viewport of a resident image).  The line also
checks that the window equals the same pixels of the whole image.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import avir_b200 as ab  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


class WindowInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_x0", "src_w", "src_y0", "src_h")]


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(n, ww, wh, sw=7680, sh=4320, nw=3840, nh=2160, ch=4):
    lib = ab.lib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    lib.lancirb200_plan_workspace_bytes.argtypes = [vp, vp]
    lib.lancirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    lib.lancirb200_window_query.argtypes = [vp, i, i, i, i, vp]
    lib.lancirb200_window_workspace_bytes.argtypes = [vp, i, i, i, i, vp]
    lib.lancirb200_resize_window_device.argtypes = [vp, i, i, i, i, vp, sz, vp, sz, vp, vp]
    h = ab.host_lib().lancirb200_host_desc_create(0, 0, sw, sh, nw, nh, ch, 0.0, 0.0, 0.0, 0.0, 3.0)
    assert h
    plan = C.c_void_p()
    assert lib.lancirb200_plan_create(C.c_void_p(ab.host_lib().lancirb200_host_desc_get(h)), C.byref(plan)) == 0, \
        lib.avirb200_last_error()
    g = torch.Generator(device="cuda").manual_seed(1)
    d_src = torch.randint(0, 256, (sh, sw, ch), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    d_dst = torch.zeros((nh, nw, ch), device="cuda", dtype=torch.uint8)
    wsb = C.c_size_t()
    assert lib.lancirb200_plan_workspace_bytes(plan, C.byref(wsb)) == 0
    d_ws = torch.empty(wsb.value, dtype=torch.uint8, device="cuda")
    win = ((nw - ww) // 2 + 1, (nh - wh) // 2 + 1, ww, wh)  # centred, at odd offsets
    fi, wn = WindowInfo(), C.c_size_t()
    assert lib.lancirb200_window_query(plan, *win, C.byref(fi)) == 0, lib.avirb200_last_error()
    assert lib.lancirb200_window_workspace_bytes(plan, *win, C.byref(wn)) == 0
    w_dst = torch.zeros((wh, ww, ch), device="cuda", dtype=torch.uint8)
    w_ws = torch.empty(wn.value, dtype=torch.uint8, device="cuda")
    w_src = d_src.data_ptr() + (fi.src_y0 * sw + fi.src_x0) * ch
    st = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def full():
        assert lib.lancirb200_resize_device(plan, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch,
                                            d_ws.data_ptr(), st) == 0

    def window():
        assert lib.lancirb200_resize_window_device(plan, *win, w_src, sw * ch, w_dst.data_ptr(), ww * ch,
                                                   w_ws.data_ptr(), st) == 0

    def timed(fn):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(3):
        full()
        window()
    tf, tw = [], []
    for _ in range(n):  # alternated
        tf.append(timed(full))
        tw.append(timed(window))
    torch.cuda.synchronize()
    x0, y0 = win[0], win[1]
    same = bool(torch.equal(w_dst, d_dst[y0:y0 + wh, x0:x0 + ww]))
    fms, wms = sorted(tf)[n // 2], sorted(tw)[n // 2]
    mid_b = 4 * ch  # intermediate bytes per pixel (float)
    full_bytes = sw * sh * ch + 2 * nh * sw * mid_b + nw * nh * ch
    win_bytes = fi.src_w * fi.src_h * ch + 2 * wh * fi.src_w * mid_b + ww * wh * ch
    rec = {"geometry": "%dx%d->%dx%d RGBA u8, la 3" % (sw, sh, nw, nh), "window": list(win),
           "footprint": [fi.src_x0, fi.src_w, fi.src_y0, fi.src_h],
           "window_bytes_equal_full_crop": same, "n": n,
           "full_ms": round(fms, 4), "window_ms": round(wms, 4), "window_over_full": round(wms / fms, 4),
           "full_bytes": full_bytes, "window_bytes": win_bytes, "bytes_ratio": round(win_bytes / full_bytes, 4),
           "full_hbm_share": round(full_bytes / (fms * 1e-3) / HBM_BPS, 3),
           "window_hbm_share": round(win_bytes / (wms * 1e-3) / HBM_BPS, 3),
           "full_ms_spread": [round(min(tf), 4), round(max(tf), 4)],
           "window_ms_spread": [round(min(tw), 4), round(max(tw), 4)],
           "workspace_bytes": [wsb.value, wn.value]}
    lib.lancirb200_plan_destroy(plan)
    ab.host_lib().lancirb200_host_desc_free(h)
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
