#!/usr/bin/env python
"""Device time of avirb200_resize_device against avirb200_resize_sharded_local at 2 and 8 bands on one GPU,
for an error-diffused cfg5 (7680x4320 -> 1920x1080 RGBA u8, sRGB gamma, fpclass_float8_dil with
CImageResizerDithererErrdDIL) and a cfg3 on double buffers (7680x4320 -> 3840x2160 RGBA f64 -> f64), and the
error-diffusion kernel's share of each call's kernel time (torch.profiler).  CUDA events, L2 flushed before
every call, 3 warm-ups, the calls alternated, median of N.

    python profiles/sharded_errd_times.py [--n 20]

Each sharded result is checked against resize_device's bytes first.  On one GPU the bands run one after
another: the numbers show the cost of banding (casts and ditherer per band), not multi-GPU scaling.
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
import cases as cs  # noqa: E402

CASES = {
    "cfg5-errd": (5, 7680, 4320, 1920, 1080, 4, np.uint8, np.uint8, 8, {"gamma": True, "alpha": 3}),
    "cfg3-f64": (2, 7680, 4320, 3840, 2160, 4, np.float64, np.float64, 16, {}),
}
TT = {np.dtype(np.uint8): torch.uint8, np.dtype(np.float64): torch.float64}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20)
    a = ap.parse_args()
    L = ab.lib()
    vp, sz = C.c_void_p, C.c_size_t
    L.avirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    L.avirb200_resize_sharded_local.argtypes = [vp, C.c_int, vp, sz, vp, sz, vp, vp]
    L.avirb200_shard_workspace_bytes.argtypes = [vp, C.c_int, C.c_int, vp]
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for name, case in CASES.items():
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        g = torch.Generator(device="cuda").manual_seed(5)
        if np.dtype(ti).kind == "f":
            src = torch.rand((sh, sw, ch), generator=g, device="cuda", dtype=torch.float64)
        else:
            src = torch.randint(0, 256, (sh, sw, ch), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
        rs, v = cs.resizer_and_vars(case)
        h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, v)
        pl = C.c_void_p()
        assert L.avirb200_plan_create(C.c_void_p(dp), C.byref(pl)) == 0, L.avirb200_last_error()
        wsf = C.c_size_t()
        L.avirb200_plan_workspace_bytes(pl, C.byref(wsf))
        nbytes = wsf.value
        for k in (2, 8):
            nbytes = max(nbytes, sum(_shard_ws(L, pl, r, k) for r in range(k)))
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        dst = torch.empty((nh, nw, ch), dtype=TT[np.dtype(to)], device="cuda")
        calls = {"device": lambda: L.avirb200_resize_device(pl, src.data_ptr(), sw * ch, dst.data_ptr(), nw * ch,
                                                            ws.data_ptr(), None)}
        for k in (2, 8):
            calls["sharded_local-%d" % k] = (lambda k=k: L.avirb200_resize_sharded_local(
                pl, k, src.data_ptr(), sw * ch, dst.data_ptr(), nw * ch, ws.data_ptr(), None))
        assert calls["device"]() == 0
        torch.cuda.synchronize()
        ref = dst.clone()
        for key, fn in calls.items():
            dst.zero_()
            assert fn() == 0, L.avirb200_last_error()
            torch.cuda.synchronize()
            assert torch.equal(dst.view(torch.uint8), ref.view(torch.uint8)), (name, key)
        times = {key: [] for key in calls}
        for it in range(3 + a.n):
            for key, fn in calls.items():
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                if it >= 3:
                    times[key].append(e0.elapsed_time(e1))
        shares = {}
        for key, fn in calls.items():
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fn()
                torch.cuda.synchronize()
            tot = errd = 0.0
            for ev in prof.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA:
                    tot += ev.device_time
                    if "errd_kernel" in ev.name:
                        errd += ev.device_time
            shares[key] = round(errd / tot, 3) if tot > 0 else None
        for key in calls:
            t = np.array(times[key])
            print(json.dumps({"case": name, "call": key, "median_ms": round(float(np.median(t)), 4),
                              "min_ms": round(float(t.min()), 4), "max_ms": round(float(t.max()), 4),
                              "errd_kernel_share": shares[key]}), flush=True)
        L.avirb200_plan_destroy(pl)
        rs.free_descriptor(h)


def _shard_ws(L, pl, r, k):
    b = C.c_size_t()
    assert L.avirb200_shard_workspace_bytes(pl, r, k, C.byref(b)) == 0
    return b.value


if __name__ == "__main__":
    main()
