"""Images past 16- and 32-bit extents on the GPU (run with -m gpu on an H100).

Two kinds of limit a kernel can trip over without any small or full-size 8K test noticing:

* 16-bit extents.  A launch has at most 65535 blocks along y.  The generic kernel puts blocks of lines
  there: a 4-channel pass whose outputs each read thousands of source positions gets one line per
  block, so a 66000-column image needs 66000 of them, and a tall strip at 16 lines per block needs
  them past 1 048 560 rows.  The tall and wide cases below run every kernel family and CLancIR past 65535
  rows or columns, against upstream (oracle/_ref, threaded) or, where it is absent, the C port.
* 32-bit offsets.  Sources past 2^32 bytes, intermediates past 2^31 floats, destinations past 2^32
  bytes, the widen / narrow and double cast kernels past 2^31 elements, the ditherer past 2 GiB.  One
  missed 64-bit product would corrupt only the rows beyond the limit.  The oracle is window tiling: the
  destination is cut into tiles whose every buffer (footprint source, intermediate, output) stays far
  below 2^31 bytes, each tile's footprint is copied into a small tensor of its own and resized with the
  window call, and the big call's crop must equal it bit for bit, the tiles covering every destination
  element.  The window tests pin windows to upstream on small images, so a mismatch here can only come
  from offset arithmetic.  Error-diffusion plans refuse windows: that case is compared with upstream.

Sources are generated on the device from a seeded generator.  Every case checks the free device memory
first and skips, with the need in the message, when another tenant holds too much of it; no case needs
more than about 20 GB, and each frees its buffers before the next.  The host-buffer entry points run in
a child process, so that the library's device staging for a > 4 GiB image (kept for the next host
call) does not outlive them.  Peak device memory and time per case: profiles/h100_extents.txt."""
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_gpu_layouts import _ok, avir_plan, plan_workspace

pytestmark = pytest.mark.gpu

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GiB = 1 << 30
MARGIN = 2 * GiB          # free device memory a case leaves to other tenants beyond its own need
REF_THREADS = max(1, min(os.cpu_count() or 1, 32))
FAMILY_IDS = {0: "product", 2: "tile", 1: "generic"}

# ---- tall and wide images: past 65535 lines ------------------------------------------------------------

# The generic kernel at one line per block (one output reads 6600 source positions; the tile kernel declines
# the footprint): 66000 columns of the column pass, 66000 rows of the row pass.
LPB1_COL = (1, 66000, 6600, 66000, 2, 4, u8, u8, 8, {})
LPB1_ROW = (1, 6600, 66000, 2, 66000, 4, u8, u8, 8, {})
# A generic-only chain (filtered upsample, build mode 0, k < 2) at 16 lines per block: 68750 blocks of rows.
STRIP = (1, 4, 1100000, 6, 1650000, 4, u8, u8, 8, {"buildmode": 0})
TALL = {
    "lpb1-col": LPB1_COL,
    "lpb1-row": LPB1_ROW,
    "strip-1.1M": STRIP,
    "stream-tall": (2, 64, 140000, 32, 70000, 4, f32, f32, 16, {}),         # the k = 2 chain
    "stream-wide": (2, 140000, 64, 70000, 32, 4, f32, f32, 16, {}),
    "tile-tall": (1, 96, 100000, 64, 66667, 4, u8, u8, 8, {}),              # ratio 1.5: the tile kernel
    "tile-wide": (1, 100000, 96, 66667, 64, 4, u8, u8, 8, {}),
    "gray-tall": (1, 64, 140000, 32, 70000, 1, f32, f32, 16, {}),           # widened to 4 channels
    "rgb-wide": (0, 140000, 48, 70000, 24, 3, u8, u8, 8, {}),
}
# avirb200_plan_kernel_paths of each tall case (bit 0 / 1: row / column pass on the streaming kernel, bit 2 / 3:
# on the tile kernel; a pass with neither runs the generic kernel): the pass under test must not quietly move
# to another family when a routing rule changes.  The packed whole-image calls take the first family that
# applies, in the product order.
TALL_PATHS = {
    "lpb1-col": lambda m: m & 0b1010 == 0,        # column pass: generic
    "lpb1-row": lambda m: m & 0b0101 == 0,        # row pass: generic
    "strip-1.1M": lambda m: m == 0,               # both passes generic
    "stream-tall": lambda m: m & 0b11 == 0b11,
    "stream-wide": lambda m: m & 0b11 == 0b11,
    "tile-tall": lambda m: m == 0b1100,
    "tile-wide": lambda m: m == 0b1100,
    "gray-tall": lambda m: m & 0b11 == 0b11,      # widened onto the streaming kernel
    "rgb-wide": lambda m: m != 0,                 # widened onto the 4-channel kernels
}
# CLancIR: (src_w, src_h, dst_w, dst_h, channels, type); destinations keep to 65535 rows (its documented bound)
LANCIR_TALL = {
    "lancir-tall": (64, 140000, 48, 60000, 4, u8),
    "lancir-wide": (140000, 64, 100000, 48, 4, u8),
    "lancir-tall-rgb": (48, 100000, 40, 65535, 3, f32),
}

# ---- offsets past 32 bits --------------------------------------------------------------------------------

BIG = {
    # source bytes 4.36e9, intermediate 2.18e9 floats
    "headline-u8": (2, 33000, 33000, 16500, 16500, 4, u8, u8, 8, {}),
    # source elements 2.15e9 (8.6 GB)
    "dil-f32": (2, 23200, 23200, 11600, 11600, 4, f32, f32, 16, {}),
    # destination bytes 4.36e9
    "cfg2-up": (1, 16500, 16500, 33000, 33000, 4, u8, u8, 8, {}),
    # the cfg4 chain on a 5.2 GB source
    "cfg4": (1, 32768, 20000, 8192, 5000, 4, u16, u16, 16, {}),
    # a non-integer ratio: the tile kernel; source 4.36e9 bytes, intermediate 2.9e9 floats
    "tile-1.5": (1, 33000, 33000, 22000, 22000, 4, u8, u8, 8, {}),
    # widen past 2^31 elements (2.19e9 source elements)
    "rgb-down": (0, 27000, 27000, 13500, 13500, 3, u8, u8, 8, {}),
    # narrow past 2^31 elements (2.19e9 destination elements)
    "rgb-up": (0, 13500, 13500, 27000, 27000, 3, u8, u8, 8, {}),
    # a double source of 4.3e9 bytes: narrow_f64_kernel; double destination through widen_f32_kernel
    "f64": (1, 16384, 8192, 8192, 4096, 4, f64, f64, 16, {}),
}
# the kernel families each big case runs on (every family crosses each limit on the headline and cfg2 cases)
BIG_RUNS = [(n, fam) for n in BIG for fam in ((0, 2, 1) if n in ("headline-u8", "cfg2-up") else (0,))]
# error diffusion with a u16 destination of 2.18e9 bytes, 500 row groups
ERRD_BIG = (4, 8500, 8000, 17000, 16000, 4, u16, u16, 16, {})
LANCIR_BIG = (33000, 33000, 16500, 16500, 4, u8)    # the intermediate: 2.18e9 floats
LANCIR_SHARD = (33000, 33000, 4125, 4125, 4, u8)    # band offsets into a 4.36e9-byte source
TILES_PER_AXIS = 6
WINDOW_LIMIT = 1 << 31   # every buffer of a tile's window call stays below this many bytes


def tiles(nw, nh, n=TILES_PER_AXIS):
    """The destination cut into n x n windows (x0, y0, w, h), edge tiles taking the remainder."""
    tw, th = -(-nw // n), -(-nh // n)
    return [(x, y, min(tw, nw - x), min(th, nh - y)) for y in range(0, nh, th) for x in range(0, nw, tw)]


def tile_buffers(fi, win, ch, ti, to):
    """Bytes of a window call's footprint source, intermediate (at most 4 float lanes a pixel, footprint rows x
    window columns for AVIR, window rows x footprint columns for CLancIR) and destination."""
    return (fi.src_w * fi.src_h * ch * np.dtype(ti).itemsize, max(fi.src_h * win[2], win[3] * fi.src_w) * 4 * 4,
            win[2] * win[3] * ch * np.dtype(to).itemsize)


# ---- helpers ---------------------------------------------------------------------------------------------

def torch_type(dt):
    import torch
    return {np.dtype(u8): torch.uint8, np.dtype(u16): torch.uint16, np.dtype(f32): torch.float32,
            np.dtype(f64): torch.float64}[np.dtype(dt)]


def device_image(n, dt, seed):
    """n elements of type dt on the device from a seeded generator, in chunks (no int32 temporary of
    the whole image): integers uniform over the type's range, floats uniform in [0, 1)."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty(n, dtype=torch_type(dt), device="cuda")
    step = 1 << 28
    for a in range(0, n, step):
        m = min(step, n - a)
        if np.dtype(dt).kind == "f":
            out[a:a + m] = torch.rand(m, generator=g, device="cuda", dtype=torch_type(dt))
        else:
            hi = np.iinfo(dt).max + 1
            out[a:a + m] = torch.randint(0, hi, (m,), generator=g, device="cuda", dtype=torch.int32).to(torch_type(dt))
    return out


def need_device(nbytes, what):
    """Skips (with the numbers) unless the device has nbytes free plus MARGIN for other tenants."""
    import torch
    free, total = torch.cuda.mem_get_info()
    if free < nbytes + MARGIN:
        pytest.skip("%s needs %.1f GB of device memory plus %.0f GB margin; %.1f GB of %.1f GB free"
                    % (what, nbytes / 1e9, MARGIN / 1e9, free / 1e9, total / 1e9))


def release():
    import gc
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def mismatching_elements(a, b, esize):
    """Elements whose bytes differ between two byte tensors of equal shape (last axis: elements x esize)."""
    assert a.shape == b.shape
    d = (a != b)
    return int(d.reshape(*d.shape[:-1], -1, esize).any(-1).sum().item())


class Record:
    """Time and peak device memory of a case, printed as one line (-s) and appended to the file that
    AVIRB200_EXTENTS_LOG names, if any."""

    def __init__(self, name):
        import torch
        self.name, self.t0 = name, time.perf_counter()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        self.notes = []

    def done(self, **kw):
        import torch
        torch.cuda.synchronize()
        line = dict(case=self.name, seconds=round(time.perf_counter() - self.t0, 2),
                    peak_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2), **kw)
        print("extents:", json.dumps(line))
        path = os.environ.get("AVIRB200_EXTENTS_LOG")
        if path:
            with open(path, "a") as f:
                f.write(json.dumps(line) + "\n")


def reference(case, src):
    """Upstream (threaded) where oracle/_ref is built, else the C port."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    if o.have_ref():
        return o.ref_resize(src, nw, nh, to, fpclass=fp, resbits=rb, nthreads=REF_THREADS, **cs.ref_kwargs(kw))
    return cs.port_output(case, src)[0]


def device_resize(L, pl, case, d_src, ws=None):
    """avirb200_resize_device on packed buffers: the destination as a byte tensor (nh, nw * ch * size)."""
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    d_dst = torch.empty((nh, nw * ch * np.dtype(to).itemsize), dtype=torch.uint8, device="cuda")
    if ws is None:
        ws = torch.empty(max(plan_workspace(L, pl), 1), dtype=torch.uint8, device="cuda")
    _ok(L.avirb200_resize_device(pl, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch, ws.data_ptr(), None))
    torch.cuda.synchronize()
    return d_dst


# ---- tall and wide ---------------------------------------------------------------------------------------

_tall_ref = {}


@pytest.mark.parametrize("family", [0, 2, 1], ids=["product", "tile", "generic"])
@pytest.mark.parametrize("name", list(TALL))
def test_tall_and_wide_images(name, family):
    import torch
    case = TALL[name]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    if name not in _tall_ref:   # (one source and reference for the three families)
        _tall_ref.clear()
        src = cs.make_input(case, seed=17)
        t0 = time.perf_counter()
        _tall_ref[name] = (src, reference(case, src), time.perf_counter() - t0)
    src, want, ref_s = _tall_ref[name]
    with avir_plan(case, family) as (L, pl):
        need_device(src.nbytes + want.nbytes + plan_workspace(L, pl), name)
        rec = Record("%s/%s" % (name, FAMILY_IDS[family]))
        d_src = torch.from_numpy(src.reshape(-1).view(np.uint8)).cuda()
        got = device_resize(L, pl, case, d_src).cpu().numpy().view(to).reshape(nh, nw, ch)
        bad = cs.count_mismatch(want, got)
        paths = L.avirb200_plan_kernel_paths(pl)
        widened = plan_workspace(L, pl) >= nw * sh * 4 * 4
        rec.done(mismatches=bad, kernel_paths=paths, reference="upstream" if o.have_ref() else "port",
                 reference_seconds=round(ref_s, 2))
    del d_src
    release()
    assert bad == 0
    assert TALL_PATHS[name](paths), bin(paths)
    assert widened or ch == 4


_lancir_ref = {}


@pytest.mark.parametrize("name", list(LANCIR_TALL))
def test_lancir_tall_and_wide_images(name):
    import torch
    from test_gpu_lancir_window import lancir_plan
    sw, sh, nw, nh, ch, ti = LANCIR_TALL[name]
    src = o.lcg_image(sh, sw, ch, ti, seed=19)
    with lancir_plan(sw, sh, nw, nh, ch, ti, ti, {}) as (L, pl, dp):
        t0 = time.perf_counter()
        if o.have_ref():
            r, want = o.lancir_ref(src, nw, nh, ti)
            assert r == nh
        else:
            want = np.zeros((nh, nw, ch), ti)
            assert cs.port().lancir_port_resize(dp, src.ctypes.data, sw * ch, want.ctypes.data, nw * ch) == 0
        ref_s = time.perf_counter() - t0
        n = C.c_size_t()
        _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
        need_device(src.nbytes + want.nbytes + n.value, name)
        rec = Record(name)
        d_src = torch.from_numpy(src.reshape(-1).view(np.uint8)).cuda()
        d_dst = torch.empty(want.nbytes, dtype=torch.uint8, device="cuda")
        ws = torch.empty(max(n.value, 1), dtype=torch.uint8, device="cuda")
        _ok(L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, d_dst.data_ptr(), nw * ch, ws.data_ptr(), None))
        got = d_dst.cpu().numpy().view(ti).reshape(nh, nw, ch)
        bad = cs.count_mismatch(want, got)
        rec.done(mismatches=bad, reference="upstream" if o.have_ref() else "port", reference_seconds=round(ref_s, 2))
    del d_src, d_dst, ws
    release()
    assert bad == 0


# ---- offsets past 32 bits: window tiling ----------------------------------------------------------------

def check_tiles(name, d_dst, d_src, case, query, window, ws_bytes):
    """Every tile of the destination through the window call on a copy of its footprint alone, against the
    big call's crop: (mismatching elements, tiles, largest tile buffer in bytes)."""
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    es, eo = np.dtype(ti).itemsize, np.dtype(to).itemsize
    src2d = d_src.view(torch.uint8).reshape(sh, sw * ch * es)
    covered = torch.zeros((nh, nw), dtype=torch.int32, device="cuda")
    bad, largest, wins = 0, 0, tiles(nw, nh)
    for win in wins:
        x0, y0, w, h = win
        fi = query(win)
        bufs = tile_buffers(fi, win, ch, ti, to)
        largest = max(largest, max(bufs))
        assert max(bufs) < WINDOW_LIMIT // 2, (name, win, bufs)
        foot = src2d[fi.src_y0:fi.src_y0 + fi.src_h, fi.src_x0 * ch * es:(fi.src_x0 + fi.src_w) * ch * es].contiguous()
        out = torch.empty((h, w * ch * eo), dtype=torch.uint8, device="cuda")
        ws = torch.empty(max(ws_bytes(win), 1), dtype=torch.uint8, device="cuda")
        window(win, foot.data_ptr(), fi.src_w * ch, out.data_ptr(), w * ch, ws.data_ptr())
        torch.cuda.synchronize()
        bad += mismatching_elements(d_dst[y0:y0 + h, x0 * ch * eo:(x0 + w) * ch * eo], out, eo)
        covered[y0:y0 + h, x0:x0 + w] += 1
        del foot, out, ws
    assert int((covered != 1).sum().item()) == 0, "the tiles do not cover the destination exactly once"
    return bad, len(wins), largest


def avir_tiles(L, pl, name, case, d_src, d_dst):
    from test_gpu_window import query, wlib
    L = wlib()

    def window(win, src, sp, dst, dp, ws):
        _ok(L.avirb200_resize_window_device(pl, *win, src, sp, dst, dp, ws, None))

    return check_tiles(name, d_dst, d_src, case, lambda win: query(L, pl, win)[0], window,
                       lambda win: query(L, pl, win)[1])


def big_need(case, ws):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    return sw * sh * ch * np.dtype(ti).itemsize + nw * nh * ch * np.dtype(to).itemsize + ws + GiB


@pytest.mark.parametrize("name,family", BIG_RUNS, ids=["%s-%s" % (n, FAMILY_IDS[f]) for n, f in BIG_RUNS])
def test_offsets_past_32_bits(name, family):
    case = BIG[name]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    with avir_plan(case, family) as (L, pl):
        n = plan_workspace(L, pl)
        need_device(big_need(case, n), name)
        rec = Record("%s/%s" % (name, FAMILY_IDS[family]))
        d_src = device_image(sh * sw * ch, ti, seed=23)
        d_dst = device_resize(L, pl, case, d_src)
        bad, ntiles, largest = avir_tiles(L, pl, name, case, d_src, d_dst)
        rec.done(mismatches=bad, tiles=ntiles, largest_tile_buffer_mb=round(largest / 1e6, 1),
                 workspace_gb=round(n / 1e9, 2))
        del d_src, d_dst
    release()
    assert bad == 0


def test_headline_offsets_against_upstream():
    """The headline case in full against threaded upstream, where the host has the memory for it."""
    import torch
    case = BIG["headline-u8"]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    if not o.have_ref():
        pytest.skip("oracle/_ref not built: upstream is not available")
    host_need = 2 * (sw * sh * ch + nw * nh * ch) + 4 * GiB
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail < host_need:
        pytest.skip("upstream on 33000^2 RGBA needs %.1f GB of host memory; %.1f GB available"
                    % (host_need / 1e9, avail / 1e9))
    with avir_plan(case, 0) as (L, pl):
        need_device(big_need(case, plan_workspace(L, pl)), "headline-u8")
        rec = Record("headline-u8/upstream")
        d_src = device_image(sh * sw * ch, ti, seed=29)
        got = device_resize(L, pl, case, d_src).cpu().numpy().reshape(nh, nw, ch)
        src = d_src.cpu().numpy().reshape(sh, sw, ch)
        del d_src
        release()
        t0 = time.perf_counter()
        want = o.ref_resize(src, nw, nh, to, fpclass=fp, resbits=rb, nthreads=REF_THREADS, **cs.ref_kwargs(kw))
        ref_s = time.perf_counter() - t0
        bad = cs.count_mismatch(want, got)
        rec.done(mismatches=bad, reference_seconds=round(ref_s, 1), reference_threads=REF_THREADS)
    assert bad == 0


def test_error_diffusion_past_2_gib_against_upstream():
    """errd_kernel storing a u16 destination of 2.18e9 bytes (500 row groups, every block resident): windows
    refuse error diffusion, so the whole image is compared with upstream (or the port)."""
    import torch
    case = ERRD_BIG
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    assert (nh + 31) // 32 <= 600 and nw * nh * ch * 2 > (1 << 31)
    with avir_plan(case, 0) as (L, pl):
        need_device(big_need(case, plan_workspace(L, pl)), "errd-u16")
        rec = Record("errd-u16")
        d_src = device_image(sh * sw * ch, ti, seed=31)
        got = device_resize(L, pl, case, d_src).cpu().numpy().view(to).reshape(nh, nw, ch)
        src = d_src.cpu().numpy().reshape(sh, sw, ch)
        del d_src
        release()
        t0 = time.perf_counter()
        want = reference(case, src)
        ref_s = time.perf_counter() - t0
        bad = cs.count_mismatch(want, got)
        rec.done(mismatches=bad, reference="upstream" if o.have_ref() else "port", reference_seconds=round(ref_s, 1),
                 reference_threads=REF_THREADS)
    assert bad == 0


def test_entry_points_past_4_gib():
    """The headline case through the per-pass pair, the sharded schedule on one device (3 bands, the halo
    fused into the kernels and moved by device copies) and a window whose source pointer lies past 4 GiB
    into the whole image, each against avirb200_resize_device."""
    import torch
    case = BIG["headline-u8"]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    with avir_plan(case, 0) as (L, pl):
        L.avirb200_shard_workspace_bytes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        sizes = []
        for r in range(3):
            b = C.c_size_t()
            _ok(L.avirb200_shard_workspace_bytes(pl, r, 3, C.byref(b)))
            sizes.append(b.value)
        n = max(plan_workspace(L, pl), sum(sizes))
        need_device(big_need(case, n) + nw * nh * ch, "headline entry points")
        rec = Record("headline-u8/entry-points")
        d_src = device_image(sh * sw * ch, ti, seed=37)
        ws = torch.empty(n, dtype=torch.uint8, device="cuda")
        want = device_resize(L, pl, case, d_src, ws)
        got = torch.empty_like(want)
        results = {}
        # the per-pass pair
        got.fill_(0xA5)
        _ok(L.avirb200_row_pass_device(pl, d_src.data_ptr(), sw * ch, ws.data_ptr(), None))
        _ok(L.avirb200_col_pass_device(pl, ws.data_ptr(), got.data_ptr(), nw * ch, None))
        torch.cuda.synchronize()
        results["per-pass"] = mismatching_elements(want, got, 1)
        # three bands on this device
        for overlap in (3, 1):
            _ok(L.avirb200_plan_set_option(pl, ab.OPT_OVERLAP_HALO, overlap))
            got.fill_(0xA5)
            _ok(L.avirb200_resize_sharded_local(pl, 3, d_src.data_ptr(), sw * ch, got.data_ptr(), nw * ch,
                                                ws.data_ptr(), None))
            torch.cuda.synchronize()
            results["sharded-local-overlap%d" % overlap] = mismatching_elements(want, got, 1)
        del got, ws
        # windows whose footprint starts past 4 GiB into the source: the source pointer inside the big buffer
        from test_gpu_window import query, wlib
        Lw = wlib()
        for win in [(nw // 2 + 7, nh - 180, 3001, 179), (nw - 2048, nh - 100, 2048, 100), (1, nh - 1, nw - 1, 1)]:
            fi, wn = query(Lw, pl, win)
            off = (fi.src_y0 * sw + fi.src_x0) * ch
            assert off > (1 << 32), (win, off)
            out = torch.empty((win[3], win[2] * ch), dtype=torch.uint8, device="cuda")
            wws = torch.empty(max(wn, 1), dtype=torch.uint8, device="cuda")
            _ok(Lw.avirb200_resize_window_device(pl, *win, d_src.data_ptr() + off, sw * ch, out.data_ptr(), win[2] * ch,
                                                 wws.data_ptr(), None))
            torch.cuda.synchronize()
            x0, y0, w, h = win
            results["window-%d-%d" % (x0, y0)] = mismatching_elements(want[y0:y0 + h, x0 * ch:(x0 + w) * ch], out, 1)
            del out, wws
        rec.done(mismatches=results)
        del d_src, want
    release()
    assert all(v == 0 for v in results.values()), results


# ---- CLancIR ---------------------------------------------------------------------------------------------

def lancir_workspace(L, pl, nranks=0):
    """lancirb200_plan_workspace_bytes, or the sum of the nranks bands' lancirb200_shard_workspace_bytes."""
    L.lancirb200_shard_workspace_bytes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    b = C.c_size_t()
    if nranks == 0:
        _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(b)))
        return b.value
    total = 0
    for r in range(nranks):
        _ok(L.lancirb200_shard_workspace_bytes(pl, r, nranks, C.byref(b)))
        total += b.value
    return total


def test_lancir_offsets_past_32_bits():
    """CLancIR 33000^2 -> 16500^2 RGBA u8 (an intermediate of 2.18e9 floats): lancirb200_resize_device against
    window tiling."""
    import torch
    from test_gpu_lancir_window import lancir_plan, query
    sw, sh, nw, nh, ch, ti = LANCIR_BIG
    case = (0, sw, sh, nw, nh, ch, ti, ti, 8, {})
    with lancir_plan(sw, sh, nw, nh, ch, ti, ti, {}) as (L, pl, dp):
        n = lancir_workspace(L, pl)
        need_device(big_need(case, n), "lancir-big")
        rec = Record("lancir-u8")
        d_src = device_image(sh * sw * ch, ti, seed=41)
        ws = torch.empty(n, dtype=torch.uint8, device="cuda")
        want = torch.empty((nh, nw * ch), dtype=torch.uint8, device="cuda")
        _ok(L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, want.data_ptr(), nw * ch, ws.data_ptr(), None))
        torch.cuda.synchronize()
        del ws

        def window(win, src, sp, dst, dstp, wsp):
            _ok(L.lancirb200_resize_window_device(pl, *win, src, sp, dst, dstp, wsp, None))

        bad, ntiles, largest = check_tiles("lancir-u8", want, d_src, case, lambda win: query(L, pl, win)[0], window,
                                           lambda win: query(L, pl, win)[1])
        rec.done(mismatches=bad, tiles=ntiles, largest_tile_buffer_mb=round(largest / 1e6, 1), workspace_gb=round(n / 1e9, 2))
        del d_src, want
    release()
    assert bad == 0


def test_lancir_sharded_past_4_gib():
    """CLancIR's sharded schedule on one device (3 bands; the neighbours' source rows read in place) on a 4.36 GB
    source, against lancirb200_resize_device.  An 8x downscale keeps the bands' workspaces small."""
    import torch
    from test_gpu_lancir_window import lancir_plan
    sw, sh, nw, nh, ch, ti = LANCIR_SHARD
    case = (0, sw, sh, nw, nh, ch, ti, ti, 8, {})
    with lancir_plan(sw, sh, nw, nh, ch, ti, ti, {}) as (L, pl, dp):
        L.lancirb200_resize_sharded_local.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p,
                                                      C.c_size_t, C.c_void_p, C.c_void_p]
        n = max(lancir_workspace(L, pl), lancir_workspace(L, pl, 3))
        need_device(big_need(case, n) + nw * nh * ch, "lancir sharded")
        rec = Record("lancir-u8/sharded-local")
        d_src = device_image(sh * sw * ch, ti, seed=47)
        ws = torch.empty(n, dtype=torch.uint8, device="cuda")
        want = torch.empty((nh, nw * ch), dtype=torch.uint8, device="cuda")
        _ok(L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, want.data_ptr(), nw * ch, ws.data_ptr(), None))
        got = torch.full_like(want, 0xA5)
        _ok(L.lancirb200_resize_sharded_local(pl, 3, d_src.data_ptr(), sw * ch, got.data_ptr(), nw * ch, ws.data_ptr(),
                                              None))
        torch.cuda.synchronize()
        bad = mismatching_elements(want, got, 1)
        rec.done(mismatches=bad, workspace_gb=round(n / 1e9, 2))
        del d_src, ws, want, got
    release()
    assert bad == 0


# ---- host buffers: a > 4 GiB pageable source, in a child process ---------------------------------------------

def host_worker(kind):
    """Child process: (mismatching elements, seconds) of the host call on a pageable source of the big headline
    image against the device call on the same pixels; the library's device staging dies with the process."""
    import torch
    if kind == "avir":
        case = BIG["headline-u8"]
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    else:
        sw, sh, nw, nh, ch, ti = LANCIR_BIG
    d_src = device_image(sh * sw * ch, u8, seed=43)
    src = d_src.cpu().numpy()              # pageable
    dst = np.full(nh * nw * ch, 0xA5, u8)  # pageable
    if kind == "avir":
        with avir_plan(case, 0) as (L, pl):
            want = device_resize(L, pl, case, d_src).cpu().numpy().reshape(-1)
            del d_src
            release()
            t0 = time.perf_counter()
            _ok(L.avirb200_resize_host(pl, src.ctypes.data, sw * ch, dst.ctypes.data, nw * ch))
    else:
        from test_gpu_lancir_window import lancir_plan
        with lancir_plan(sw, sh, nw, nh, ch, ti, ti, {}) as (L, pl, dp):
            L.lancirb200_resize_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
            b = C.c_size_t()
            _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(b)))
            ws = torch.empty(b.value, dtype=torch.uint8, device="cuda")
            out = torch.empty(nh * nw * ch, dtype=torch.uint8, device="cuda")
            _ok(L.lancirb200_resize_device(pl, d_src.data_ptr(), sw * ch, out.data_ptr(), nw * ch, ws.data_ptr(), None))
            want = out.cpu().numpy()
            del d_src, ws, out
            release()
            t0 = time.perf_counter()
            _ok(L.lancirb200_resize_host(pl, src.ctypes.data, sw * ch, dst.ctypes.data, nw * ch))
    secs = time.perf_counter() - t0
    return {"mismatches": int((want != dst).sum()), "host_call_seconds": round(secs, 2),
            "peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}


@pytest.mark.parametrize("kind", ["avir", "lancir"])
def test_host_call_on_a_pageable_source_past_4_gib(kind):
    import torch
    sw, sh, ch = 33000, 33000, 4
    # the device call's buffers, then (freed first) the library's staging: source, destination, intermediate
    need_device(sw * sh * ch + (sw // 2) * (sh // 2) * ch + sh * (sw // 2) * ch * 4 + GiB, "host call")
    host_need = 2 * sw * sh * ch + 4 * GiB
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail < host_need:
        pytest.skip("a 4.4 GB pageable source needs %.1f GB of host memory; %.1f GB available" % (host_need / 1e9, avail / 1e9))
    rec = Record("host-%s" % kind)
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_extents as t; "
            "print(json.dumps(t.host_worker(%r)))" % (ROOT, os.path.join(ROOT, "tests"), kind))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    rec.done(child=res)
    assert res["mismatches"] == 0, res
