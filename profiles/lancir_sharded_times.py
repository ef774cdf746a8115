#!/usr/bin/env python
"""Device time of row-sharded CLancIR on bench's CLancIR workload, 7680x4320 -> 3840x2160 RGBA u8 (k = 2,
12 taps per axis): lancirb200_resize_device against lancirb200_resize_sharded_local at 2 and 8 bands, every
band on this GPU, on the mailbox schedule (3) and on schedule 0 (the bands' kernels without the push and the
flag waits).  CUDA events around each call, L2 flushed before every call, calls of the variants alternated,
3 warm-ups, median and spread (min, max) of N.  Each line also checks that the sharded result equals the
whole image byte for byte.

    python profiles/lancir_sharded_times.py [--n 30]

The first line names the card, its power limit and the GPUs visible.  Strong scaling of
lancirb200_resize_sharded across GPUs is not timed here.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import avir_b200 as ab  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(n, bands=(2, 8), sw=7680, sh=4320, nw=3840, nh=2160, ch=4):
    """Variants: 0 the whole image, k > 0 k bands on the mailbox schedule, -k k bands on schedule 0 (device
    copies into the halo segments before the column passes, no flags: the bands' kernels alone)."""
    lib = ab.lib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    lib.lancirb200_plan_workspace_bytes.argtypes = [vp, vp]
    lib.lancirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    lib.lancirb200_shard_workspace_bytes.argtypes = [vp, i, i, vp]
    lib.lancirb200_resize_sharded_local.argtypes = [vp, i, vp, sz, vp, sz, vp, vp]
    lib.lancirb200_plan_set_option.argtypes = [vp, i, i]
    h = ab.host_lib().lancirb200_host_desc_create(0, 0, sw, sh, nw, nh, ch, 0.0, 0.0, 0.0, 0.0, 3.0)
    plan = C.c_void_p()
    assert lib.lancirb200_plan_create(C.c_void_p(ab.host_lib().lancirb200_host_desc_get(h)), C.byref(plan)) == 0, \
        lib.avirb200_last_error()
    g = torch.Generator(device="cuda").manual_seed(1)
    d_src = torch.randint(0, 256, (sh, sw, ch), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    b = C.c_size_t()
    assert lib.lancirb200_plan_workspace_bytes(plan, C.byref(b)) == 0
    ws_full = torch.empty(b.value, dtype=torch.uint8, device="cuda")
    ws = {}
    for k in bands:
        total = 0
        for r in range(k):
            assert lib.lancirb200_shard_workspace_bytes(plan, r, k, C.byref(b)) == 0, lib.avirb200_last_error()
            total += b.value
        ws[k] = torch.empty(total, dtype=torch.uint8, device="cuda")
    order = (0,) + tuple(bands) + tuple(-k for k in bands)
    dst = {v: torch.zeros((nh, nw, ch), device="cuda", dtype=torch.uint8) for v in order}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call(v):
        if v == 0:
            return lib.lancirb200_resize_device(plan, d_src.data_ptr(), sw * ch, dst[0].data_ptr(), nw * ch,
                                                ws_full.data_ptr(), st)
        assert lib.lancirb200_plan_set_option(plan, ab.OPT_OVERLAP_HALO, 3 if v > 0 else 0) == 0
        return lib.lancirb200_resize_sharded_local(plan, abs(v), d_src.data_ptr(), sw * ch, dst[v].data_ptr(),
                                                   nw * ch, ws[abs(v)].data_ptr(), st)

    times = {v: [] for v in order}
    for it in range(n + 3):
        for v in order:
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            assert call(v) == 0, lib.avirb200_last_error()
            e1.record()
            torch.cuda.synchronize()
            if it >= 3:
                times[v].append(e0.elapsed_time(e1))
    for v in order:
        t = times[v]
        print(json.dumps({"call": "resize_device" if v == 0 else "sharded_local", "bands": abs(v) or 1,
                          "schedule": None if v == 0 else (3 if v > 0 else 0),
                          "median_ms": round(statistics.median(t), 4), "min_ms": round(min(t), 4),
                          "max_ms": round(max(t), 4), "n": len(t),
                          "equal_to_whole_image": bool(torch.equal(dst[v], dst[0]))}), flush=True)
    lib.lancirb200_plan_destroy(plan)
    ab.host_lib().lancirb200_host_desc_free(h)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=30)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info(), "visible_gpus": torch.cuda.device_count()}), flush=True)
    run(a.n)


if __name__ == "__main__":
    main()
