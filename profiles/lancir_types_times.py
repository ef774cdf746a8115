#!/usr/bin/env python
"""Device-resident time of CLancIR per element-type pair (CUDA events, L2 flushed before every call, 3 warm-ups,
the pairs' calls alternated, median of N), with each pair's algorithmic bytes and their rate as a share of the
H100 SXM's 3.35 TB/s data-sheet HBM3 bandwidth.

    python profiles/lancir_types_times.py [--n 30] [--pairs u8-u8 u32-u32 f64-f64 u8-f64 f64-u8] [--root TREE]

Setup: 8K -> 4K RGBA (k = 2, 12 taps per axis), packed buffers (the 4-channel vector kernels).  Bytes of a
call = source read + intermediate written and read back + destination written: src + 2 x mid + dst, where mid
is dst_h x src_w pixels of floats (2 x 265.4 MB for every pair).  u8 -> u8 is the baseline, timed in the same
run.  --root times the library of another built tree (e.g. the parent commit's, u8-u8 only there); the card's
name and power limit are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HBM_BPS = 3.35e12  # H100 SXM data sheet
CODES = {"u8": 0, "u16": 1, "f32": 2, "f64": 3, "u32": 4}
SIZES = {"u8": 1, "u16": 2, "f32": 4, "f64": 8, "u32": 4}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def source(torch, t, n, g):
    """n elements of type t on the device: u8 / u32 codes of their ranges (u32: u16 codes), floats in [0, 1)."""
    if t == "u8":
        return torch.randint(0, 256, (n,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    if t == "u32":   # int32 bits of values 0..65535 are the uint32_t bits
        return torch.randint(0, 65536, (n,), generator=g, device="cuda", dtype=torch.int32)
    if t == "u16":
        return torch.randint(0, 65536, (n,), generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
    return torch.rand((n,), generator=g, device="cuda", dtype=torch.float64 if t == "f64" else torch.float32)


def run(n, pairs, sw=7680, sh=4320, nw=3840, nh=2160, ch=4):
    import torch
    import avir_b200 as ab
    lib = ab.lib()
    vp, sz = C.c_void_p, C.c_size_t
    lib.lancirb200_plan_workspace_bytes.argtypes = [vp, vp]
    lib.lancirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    g = torch.Generator(device="cuda").manual_seed(1)
    st = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    calls = []
    for pair in pairs:
        ti, to = pair.split("-")
        h = ab.host_lib().lancirb200_host_desc_create(CODES[ti], CODES[to], sw, sh, nw, nh, ch, 0.0, 0.0, 0.0, 0.0, 3.0)
        assert h, pair
        plan = C.c_void_p()
        assert lib.lancirb200_plan_create(C.c_void_p(ab.host_lib().lancirb200_host_desc_get(h)), C.byref(plan)) == 0, \
            lib.avirb200_last_error()
        wsb = C.c_size_t()
        assert lib.lancirb200_plan_workspace_bytes(plan, C.byref(wsb)) == 0
        d_src = source(torch, ti, sh * sw * ch, g)
        d_dst = torch.empty(nh * nw * ch * SIZES[to], dtype=torch.uint8, device="cuda")
        d_ws = torch.empty(wsb.value, dtype=torch.uint8, device="cuda")

        def call(plan=plan, d_src=d_src, d_dst=d_dst, d_ws=d_ws):
            assert lib.lancirb200_resize_device(plan, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch,
                                                d_ws.data_ptr(), st) == 0
        calls.append((pair, h, plan, call, (d_src, d_dst, d_ws)))

    def timed(fn):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    for _ in range(3):
        for c in calls:
            c[3]()
    times = {c[0]: [] for c in calls}
    for _ in range(n):  # alternated
        for c in calls:
            times[c[0]].append(timed(c[3]))
    torch.cuda.synchronize()
    recs = []
    mid = 2 * nh * sw * ch * 4
    for pair, h, plan, _, _ in calls:
        ti, to = pair.split("-")
        t = sorted(times[pair])
        ms = t[n // 2]
        nbytes = sw * sh * ch * SIZES[ti] + mid + nw * nh * ch * SIZES[to]
        recs.append({"pair": pair, "n": n, "ms": round(ms, 4), "ms_spread": [round(t[0], 4), round(t[-1], 4)],
                     "bytes": nbytes, "floor_ms": round(nbytes / HBM_BPS * 1e3, 4),
                     "hbm_share": round(nbytes / (ms * 1e-3) / HBM_BPS, 3)})
        lib.lancirb200_plan_destroy(plan)
        ab.host_lib().lancirb200_host_desc_free(h)
    return recs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--pairs", nargs="+", default=["u8-u8", "u32-u32", "f64-f64", "u8-f64", "f64-u8"])
    ap.add_argument("--root", default=ROOT, help="built tree whose avir_b200 package is timed")
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.root))
    print(json.dumps({"gpu": gpu_info(), "tree": "this" if os.path.abspath(a.root) == ROOT else a.root}))
    for r in run(a.n, a.pairs):
        print(json.dumps(r))


if __name__ == "__main__":
    main()
