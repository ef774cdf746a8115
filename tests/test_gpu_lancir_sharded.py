"""Row-sharded CLancIR on the GPU (run with -m gpu on an H100): lancirb200_resize_sharded_local -- every band
of an n-rank split on one device, exchanging through the same mailboxes, push and segmented column kernel as
ranks -- against lancirb200_resize_device on the whole image, byte for byte.  The multi-GPU call itself runs
in tests/lancir_sharded_worker.py under torch.distributed.run when the machine has the GPUs."""
import contextlib
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_gpu_layouts import _ok
import test_gpu_lancir_window as lw
from test_gpu_lancir_window import _geometries, _gid, full_device, window_in_place
from test_gpu_window import upload
from lancir_sharded_worker import CODE
from test_lancir_sharding import ShardInfo

pytestmark = pytest.mark.gpu

u8, u16, f32, f64, u32 = np.uint8, np.uint16, np.float32, np.float64, np.uint32
ALL_TYPES = (u8, u16, f32, f64, u32)
ERR_UNSUPPORTED = -4
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@contextlib.contextmanager
def lancir_plan(sw, sh, nw, nh, ch, ti, to, kw):
    """test_gpu_lancir_window.lancir_plan for every element type upstream's CLancIR takes."""
    h = ab.host_lib().lancirb200_host_desc_create(CODE[np.dtype(ti)], CODE[np.dtype(to)], sw, sh, nw, nh, ch,
                                                  kw.get("kx", 0.0), kw.get("ky", 0.0), kw.get("ox", 0.0),
                                                  kw.get("oy", 0.0), kw.get("la", 3.0))
    assert h
    L, pl = lw.llib(), C.c_void_p()
    dp = ab.host_lib().lancirb200_host_desc_get(h)
    try:
        _ok(L.lancirb200_plan_create(C.c_void_p(dp), C.byref(pl)))
        yield L, pl, dp
    finally:
        if pl.value:
            L.lancirb200_plan_destroy(pl)
        ab.host_lib().lancirb200_host_desc_free(h)


def slib(L):
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    L.lancirb200_shard_query.argtypes = [vp, i, i, vp]
    L.lancirb200_shard_workspace_bytes.argtypes = [vp, i, i, vp]
    L.lancirb200_resize_sharded_local.argtypes = [vp, i, vp, sz, vp, sz, vp, vp]
    L.lancirb200_resize_sharded.argtypes = [vp, vp, i, i, vp, sz, vp, sz, vp, vp]
    L.lancirb200_resize_sharded_host.argtypes = [vp, vp, i, i, vp, sz, vp, sz]
    L.lancirb200_plan_set_option.argtypes = [vp, i, i]
    return L


def splittable(L, pl, n):
    si = ShardInfo()
    for r in range(n):
        rc = L.lancirb200_shard_query(pl, r, n, C.byref(si))
        if rc != 0:
            assert rc == ERR_UNSUPPORTED
            return False
    return True


def local_ws(L, pl, n):
    import torch
    total = 0
    for r in range(n):
        b = C.c_size_t()
        _ok(L.lancirb200_shard_workspace_bytes(pl, r, n, C.byref(b)))
        total += b.value
    return torch.empty(total, dtype=torch.uint8, device="cuda")


def run_local(L, pl, d_src, src_off, src_pitch, nw, nh, ch, ti, to, n, dst_pitch=None, dst_off=0):
    """sharded_local; the source at element src_off of d_src with rows src_pitch elements apart, the destination
    likewise; returns the (nh, nw, ch) result."""
    import torch
    dst_pitch = dst_pitch or nw * ch
    eo = np.dtype(to).itemsize
    d_dst = torch.zeros((dst_off + nh * dst_pitch) * eo, dtype=torch.uint8, device="cuda")
    ws = local_ws(L, pl, n)
    _ok(L.lancirb200_resize_sharded_local(pl, n, d_src.data_ptr() + src_off * np.dtype(ti).itemsize, src_pitch,
                                          d_dst.data_ptr() + dst_off * eo, dst_pitch, ws.data_ptr(), None))
    torch.cuda.synchronize()
    out = d_dst.cpu().numpy()[dst_off * eo:].view(to).reshape(nh, dst_pitch)[:, :nw * ch]
    return np.ascontiguousarray(out).reshape(nh, nw, ch)


def same(a, b):
    return np.array_equal(a.view(np.uint8), b.view(np.uint8))


def check_local(src, nw, nh, to, kw, ranks=(2, 3, 5, 8), overlaps=(3,)):
    sh, sw, ch = src.shape
    ran = 0
    with lancir_plan(sw, sh, nw, nh, ch, src.dtype, to, kw) as (L, pl, _):
        slib(L)
        d_src = upload(src)
        full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, to)
        for ov in overlaps:
            _ok(L.lancirb200_plan_set_option(pl, ab.OPT_OVERLAP_HALO, ov))
            for n in ranks:
                if not splittable(L, pl, n):
                    continue
                ran += 1
                got = run_local(L, pl, d_src, 0, sw * ch, nw, nh, ch, src.dtype, to, n)
                assert same(full, got), (n, ov)
    return ran


# ---- the LANCIR parity geometries, 1-4 channels, 2 / 3 / 5 / 8 bands -----------------------------------------

@pytest.mark.parametrize("g", _geometries(), ids=_gid)
def test_sharded_local_equals_the_whole_image(g):
    sw, sh, nw, nh, ch, kw = g
    for c in sorted({1, 2, 3, 4} - {ch}) + [ch]:
        src = o.lcg_image(sh, sw, c, u8, seed=31 + c)
        assert check_local(src, nw, nh, u8, dict(kw)) >= 1


# ---- every element type pair on one geometry ----------------------------------------------------------------

@pytest.mark.parametrize("to", ALL_TYPES, ids=lambda t: np.dtype(t).name)
@pytest.mark.parametrize("ti", ALL_TYPES, ids=lambda t: np.dtype(t).name)
def test_type_pairs(ti, to):
    for ch in (4, 3):
        src = o.lcg_image(150, 97, ch, ti, seed=5) if ti not in (f64, u32) else \
            o.lcg_image(150, 97, ch, f32 if ti == f64 else u16, seed=5).astype(ti)
        assert check_local(src, 61, 71, to, {}, ranks=(2, 5), overlaps=(3, 0)) == 4


# ---- vector and scalar column kernels: aligned, padded and offset buffers -----------------------------------

LAYOUTS = {  # (extra source pitch, source offset, extra destination pitch, destination offset): elements
    "packed": (0, 0, 0, 0), "src-pad4": (8, 0, 4, 0), "src-pitch-not4": (6, 0, 0, 0), "src-offset1": (4, 1, 0, 0),
    "dst-odd": (0, 0, 3, 1)}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("ti", (u8, f32, f64), ids=lambda t: np.dtype(t).name)
def test_buffer_layouts(ti, layout):
    import torch
    sp, so, dp, do = LAYOUTS[layout]
    sw, sh, nw, nh, ch = 203, 177, 98, 85, 4
    src = o.lcg_image(sh, sw, ch, f32 if ti == f64 else ti, seed=7).astype(ti)
    pitch = sw * ch + sp
    back = np.zeros(so + sh * pitch + 16, ti)
    back[so:so + sh * pitch].reshape(sh, pitch)[:, :sw * ch] = src.reshape(sh, -1)
    with lancir_plan(sw, sh, nw, nh, ch, ti, u8, {}) as (L, pl, _):
        slib(L)
        full = full_device(L, pl, upload(src), sw, sh, nw, nh, ch, u8)
        d_back = upload(back)
        for ov in (3, 0):
            _ok(L.lancirb200_plan_set_option(pl, ab.OPT_OVERLAP_HALO, ov))
            for n in (2, 3, 8):
                got = run_local(L, pl, d_back, so, pitch, nw, nh, ch, ti, u8, n, nw * ch + dp, do)
                assert same(full, got), (layout, n, ov)
        assert np.array_equal(d_back.cpu().numpy(), back.view(np.uint8)), "source written"
    torch.cuda.synchronize()


# ---- asymmetric halos, one-row bands ------------------------------------------------------------------------

ASYM = [(64, 48, 103, 77, 4, u8, {}), (64, 48, 103, 77, 3, u16, {"oy": 5.5}), (64, 48, 103, 77, 4, f32, {"oy": 5.5}),
        (90, 60, 45, 30, 1, u8, {"oy": -6.5, "ky": 1.5}), (40, 30, 40, 30, 4, f32, {"oy": -2.25})]


@pytest.mark.parametrize("c", ASYM, ids=lambda c: "%dx%d-%dx%d-c%d" % c[:5] + "".join("-%s%s" % kv for kv in c[6].items()))
def test_asymmetric_halos(c):
    sw, sh, nw, nh, ch, ti, kw = c
    src = o.lcg_image(sh, sw, ch, ti, seed=11)
    with lancir_plan(sw, sh, nw, nh, ch, ti, ti, kw) as (L, pl, _):
        slib(L)
        asym = False
        for n in (2, 3, 5, 8):
            if not splittable(L, pl, n):
                continue
            for r in range(n - 1):
                a, b = ShardInfo(), ShardInfo()
                _ok(L.lancirb200_shard_query(pl, r, n, C.byref(a)))
                _ok(L.lancirb200_shard_query(pl, r + 1, n, C.byref(b)))
                asym = asym or ((a.halo_down == 0) != (b.halo_up == 0))
    if kw:
        assert asym, "no pair with rows travelling one way only"
    assert check_local(src, nw, nh, ti, kw, overlaps=(3, 0)) >= 1


def test_one_row_bands():
    """Two bands of one destination row each: a 32x downscale whose taps span the whole source, so each band
    needs every row of its neighbour's."""
    for ch, ti in ((4, u8), (3, f32), (1, u16), (4, f32)):
        src = o.lcg_image(64, 33, ch, ti, seed=12)
        assert check_local(src, 17, 2, ti, {}, ranks=(2,), overlaps=(3, 0)) == 2


# ---- full size: 8K -> 4K RGBA u8 ----------------------------------------------------------------------------

def test_full_size():
    import torch
    sw, sh, nw, nh, ch = 7680, 4320, 3840, 2160, 4
    g = torch.Generator(device="cuda").manual_seed(5)
    d_src = torch.randint(0, 256, (sh * sw * ch,), generator=g, device="cuda", dtype=torch.int32).to(torch.uint8)
    with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, _):
        slib(L)
        full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, u8)
        for ov in (3, 0):
            _ok(L.lancirb200_plan_set_option(pl, ab.OPT_OVERLAP_HALO, ov))
            for n in (2, 3, 8, 16):
                got = run_local(L, pl, d_src, 0, sw * ch, nw, nh, ch, u8, u8, n)
                assert same(full, got), (n, ov)
    del d_src
    torch.cuda.empty_cache()


# ---- a plan taller than the kernels' grid: the whole image is refused, its bands run ------------------------

def test_tall_plan():
    import torch
    sw, sh, nw, nh, ch = 6, 35000, 4, 70001, 1
    src = o.lcg_image(sh, sw, ch, u8, seed=6)
    with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, dp):
        slib(L)
        want = np.zeros((nh, nw, ch), u8)
        assert cs.port().lancir_port_resize(dp, src.ctypes.data, sw * ch, want.ctypes.data, nw * ch) == 0
        d_src = upload(src)
        n = C.c_size_t()
        _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
        buf = torch.empty(max(n.value, nh * nw * ch), dtype=torch.uint8, device="cuda")
        assert L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, buf.data_ptr(), nw * ch, buf.data_ptr(),
                                          None) == ERR_UNSUPPORTED
        wins = np.concatenate([window_in_place(L, pl, d_src, sw, ch, u8, u8, (0, 0, nw, 35000)),
                               window_in_place(L, pl, d_src, sw, ch, u8, u8, (0, 35000, nw, 35001))])
        assert same(want, wins)
        for ov in (3, 0):
            _ok(L.lancirb200_plan_set_option(pl, ab.OPT_OVERLAP_HALO, ov))
            for k in (2, 3):
                assert same(wins, run_local(L, pl, d_src, 0, sw * ch, nw, nh, ch, u8, u8, k)), (k, ov)
    torch.cuda.synchronize()


# ---- single-rank and host forms; options; errors ------------------------------------------------------------

def test_one_rank_and_host_forms():
    """nranks == 1 is lancirb200_resize_device; the host form of one rank stages through the plan's buffers."""
    import torch
    sw, sh, nw, nh, ch = 96, 54, 48, 27, 4
    src = o.lcg_image(sh, sw, ch, u8, seed=3)
    with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, _):
        slib(L)
        d_src = upload(src)
        full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, u8)
        ws = local_ws(L, pl, 1)
        d_dst = torch.zeros(nh * nw * ch, dtype=torch.uint8, device="cuda")
        _ok(L.lancirb200_resize_sharded(pl, None, 0, 1, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch,
                                        ws.data_ptr(), None))
        torch.cuda.synchronize()
        assert same(full, d_dst.cpu().numpy().reshape(nh, nw, ch))
        out = np.zeros((nh, nw, ch), u8)
        _ok(L.lancirb200_resize_sharded_host(pl, None, 0, 1, src.ctypes.data, sw * ch, out.ctypes.data, nw * ch))
        assert same(full, out)
        # (a multi-rank call needs a communicator)
        assert L.lancirb200_resize_sharded(pl, None, 0, 2, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch,
                                           ws.data_ptr(), None) == -1
        for opt, val in ((ab.OPT_OVERLAP_HALO, 1), (ab.OPT_OVERLAP_HALO, 2), (ab.OPT_KERNEL_FAMILY, 0)):
            assert L.lancirb200_plan_set_option(pl, opt, val) == -1
        assert L.lancirb200_resize_sharded_local(pl, 2, d_src.data_ptr(), sw * ch - 1, d_dst.data_ptr(), nw * ch,
                                                 ws.data_ptr(), None) == -1
        assert L.lancirb200_resize_sharded_local(pl, 28, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch,
                                                 ws.data_ptr(), None) == ERR_UNSUPPORTED


def test_consecutive_calls_with_different_sources():
    import torch
    sw, sh, nw, nh, ch = 320, 240, 160, 120, 4
    with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, _):
        slib(L)
        for seed in range(4):
            src = o.lcg_image(sh, sw, ch, u8, seed=40 + seed)
            d_src = upload(src)
            full = full_device(L, pl, d_src, sw, sh, nw, nh, ch, u8)
            assert same(full, run_local(L, pl, d_src, 0, sw * ch, nw, nh, ch, u8, u8, 3))
    torch.cuda.synchronize()


# ---- routing: vector cases run the segmented col4 kernel ----------------------------------------------------

SEG_KERNELS = ("lancir_col4_seg_kernel", "lancir_col_seg_kernel", "lancir_col4_kernel", "lancir_col_kernel",
               "lancir_row4_kernel", "lancir_row_kernel")


def routes():
    """{case: [kernels]} of one sharded_local call each, None when the profiler records no kernel activity."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    for name, ch, sp in (("vec", 4, 0), ("scalar-pitch", 4, 6), ("scalar-c3", 3, 0)):
        sw, sh, nw, nh = 96, 64, 48, 32
        src = o.lcg_image(sh, sw, ch, u8, seed=1)
        pitch = sw * ch + sp
        back = np.zeros(sh * pitch, u8)
        back.reshape(sh, pitch)[:, :sw * ch] = src.reshape(sh, -1)
        with lancir_plan(sw, sh, nw, nh, ch, u8, u8, {}) as (L, pl, _):
            slib(L)
            d_back = upload(back)
            ws = local_ws(L, pl, 2)
            d_dst = torch.zeros(nh * nw * ch, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                _ok(L.lancirb200_resize_sharded_local(pl, 2, d_back.data_ptr(), pitch, d_dst.data_ptr(), nw * ch,
                                                      ws.data_ptr(), None))
                torch.cuda.synchronize()
            evs = []
            for e in prof.events():
                for k in SEG_KERNELS:
                    if re.search(r"\b%s\b" % k, e.name):
                        evs.append((e.time_range.start, k))
                        break
            if not evs:
                return None
            out[name] = [k for _, k in sorted(evs)]
    return out


def test_sharded_local_routes_to_the_segmented_kernels():
    """Vector cases run the segmented col4 kernel on the edge rows, scalar ones the segmented scalar kernel.  Run
    in a child process: a profiler session leaves state behind in the process that runs it."""
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_lancir_sharded as t; "
            "print(json.dumps(t.routes()))" % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    if got is None:
        pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
    # per band: the plain column kernel over the interior rows, the segmented one over the edge rows, the row pass
    col4, seg4, col1, seg1 = "lancir_col4_kernel", "lancir_col4_seg_kernel", "lancir_col_kernel", "lancir_col_seg_kernel"
    assert got["vec"] == [col4, seg4, "lancir_row4_kernel"] * 2, got
    assert got["scalar-pitch"] == [col1, seg1, "lancir_row4_kernel"] * 2, got
    assert got["scalar-c3"] == [col1, seg1, "lancir_row_kernel"] * 2, got


# ---- several GPUs: lancirb200_resize_sharded, one process per GPU --------------------------------------------

def _gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_multi_gpu_sharded(nranks):
    """lancirb200_resize_sharded, mailbox (3) and NCCL (0) schedules, three calls per plan."""
    if _gpus() < nranks:
        pytest.skip("needs %d GPUs" % nranks)
    port = 29500 + (os.getpid() % 200) + nranks
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nranks),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "lancir_sharded_worker.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-4000:]
    assert "mismatches=" in r.stdout
