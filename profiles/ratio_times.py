#!/usr/bin/env python
"""Device-resident time of large-ratio resizes on each kernel family (CUDA events around
avirb200_resize_device, 3 warm-ups, median of N), with the kernels' launch configuration as the plan
reports it.  Correctness is tests/test_gpu_ratios.py's; this records what the thin layouts large ratios
need (one output per tile, few lines per block) cost, next to the product order.

    python profiles/ratio_times.py [--n 20]

One JSON line per (case, family): family product / tile / generic (plan option KERNEL_FAMILY), the
median and spread in ms, the kernel paths the plan qualifies for (avirb200_plan_kernel_paths).
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

CASES = {  # name: (fpclass, sw, sh, nw, nh, channels, type, resbits)
    "4000x3000-125x94-rgba-u8": (1, 4000, 3000, 125, 94, 4, np.uint8, 8),
    "4000x3000-125x94-rgb-u8": (1, 4000, 3000, 125, 94, 3, np.uint8, 8),
    "7680x4320-256x144-f32": (2, 7680, 4320, 256, 144, 4, np.float32, 16),
    "4032x3024-126x95-u16": (1, 4032, 3024, 126, 95, 4, np.uint16, 12),
    "2048x2048-1x1-f32": (2, 2048, 2048, 1, 1, 4, np.float32, 16),
    "6144x24-24x24-k256-u8": (1, 6144, 24, 24, 24, 4, np.uint8, 8),
    "7680x4320-3840x2160-f32": (2, 7680, 4320, 3840, 2160, 4, np.float32, 16),   # the headline ratio, for scale
}
TT = {np.uint8: torch.uint8, np.uint16: torch.uint16, np.float32: torch.float32}
FAMILIES = {"product": 0, "tile": 2, "generic": 1}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def run(name, family, n):
    fp, sw, sh, nw, nh, ch, ti, rb = CASES[name]
    lib = ab.lib()
    vp, sz = C.c_void_p, C.c_size_t
    lib.avirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    lib.avirb200_plan_set_option.argtypes = [vp, C.c_int, C.c_int]
    rs = ab.CImageResizer(rb, 0, 0, fp)
    h, dp, modes = rs.descriptor((sh, sw, ch), ti, nw, nh, ti, 0.0, ab.CImageResizerVars())
    plan = C.c_void_p()
    assert lib.avirb200_plan_create(C.c_void_p(dp), C.byref(plan)) == 0, lib.avirb200_last_error()
    assert lib.avirb200_plan_set_option(plan, ab.OPT_KERNEL_FAMILY, FAMILIES[family]) == 0
    g = torch.Generator(device="cuda").manual_seed(1)
    if ti == np.float32:
        d_src = torch.rand((sh, sw, ch), generator=g, device="cuda", dtype=torch.float32)
    else:
        top = 256 if ti == np.uint8 else 1 << rb
        d_src = torch.randint(0, top, (sh, sw, ch), generator=g, device="cuda", dtype=torch.int32).to(TT[ti])
    d_dst = torch.zeros((nh, nw, ch), device="cuda", dtype=TT[ti])
    wsb = C.c_size_t()
    assert lib.avirb200_plan_workspace_bytes(plan, C.byref(wsb)) == 0
    d_ws = torch.empty(max(wsb.value, 1), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def call():
        r = lib.avirb200_resize_device(plan, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch, d_ws.data_ptr(), st)
        assert r == 0, lib.avirb200_last_error()

    for _ in range(3):
        call()
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        call()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    rec = {"case": name, "family": family, "n": n, "ms": round(sorted(ts)[n // 2], 4),
           "ms_spread": [round(min(ts), 4), round(max(ts), 4)],
           "kernel_paths": lib.avirb200_plan_kernel_paths(plan), "build_modes": list(modes)}
    lib.avirb200_plan_destroy(plan)
    rs.free_descriptor(h)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20)
    a = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}))
    for name in CASES:
        for family in FAMILIES:
            print(json.dumps(run(name, family, a.n)), flush=True)
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
