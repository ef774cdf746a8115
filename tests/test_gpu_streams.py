"""The caller's stream, CUDA graph capture and concurrent threads on every device entry point (run with
-m gpu on an H100).

avirb200.h promises that device calls are asynchronous on the caller's stream, allocate nothing and do not
synchronise; that plans may be shared by threads and streams; and that a workspace belongs to one call in
flight.  A PyTorch caller relies on all three (side streams, CUDA graphs, data-loader threads).  Every
check below is deterministic:

* stream: on a side stream S (torch's pool streams are non-blocking: the legacy stream does not order
  against them) a bounded spin of about 0.1 s, then the real source copied over a poisoned one, then the
  call, then the destination copied out.  A kernel, memset or copy the library puts on any other stream
  runs during the spin, reads poison or leaves sentinel bytes, and the result differs every time.
  S.query() straight after the call shows that the call did not wait for S.
* graph capture: each entry point captured once on S in the global capture mode (which refuses an
  allocation or a synchronous copy anywhere in the process), replayed three times over new sources.
* threads: 8 threads on one shared plan, each with its own stream, workspace and buffers; host calls on a
  shared plan and on several plans of one device.

The reference of a call is the same call made eagerly on the legacy stream, followed by a device
synchronise; the rest of the suite proves those bit-exact against upstream, and one case per kernel family
is checked against upstream (or the C port) here as well.  Comparisons demand 0 differing elements."""
import contextlib
import ctypes as C
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
from test_gpu_lancir_window import lancir_plan, llib
from test_gpu_layouts import CFG3_DIL, F64, RGB, SHARD_CASES, TILE, _ok, avir_plan, expected, launched_kernels
from test_gpu_window import wlib
from test_lancir_window import LancirWindowInfo
from test_window import WindowInfo, crop

pytestmark = pytest.mark.gpu

u8, f32 = np.uint8, np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLEEP_CYCLES = 200_000_000  # torch.cuda._sleep: about 0.1 s at the H100's 1.98 GHz
THREADS = 8
CALLS_PER_THREAD = 4

ERRD = [(fp, 120, 80, 60, 40, 4, u8, u8, 8, {}) for fp in (3, 4, 5)]  # error diffusion of the three classes
# name: (case, kernel family, plan kernel-path bits that must be set, bits that must be clear); bits 0 / 1 =
# row / column pass on the streaming kernel, 2 / 3 = on the tile kernel (avirb200_plan_kernel_paths)
AVIR = {
    "cfg3-stream": (CFG3_DIL, 0, 0x3, 0x0),
    "tile": (TILE, 0, 0xC, 0x3),
    "tile-generic": (TILE, 1, 0xC, 0x3),   # the tile case forced onto the generic kernel
    "rgb": (RGB, 0, 0x0, 0x0),              # widened to 4 channels
    "f64": (F64, 0, 0x0, 0x0),
    "errd3": (ERRD[0], 0, 0x0, 0x0),
    "errd4": (ERRD[1], 0, 0x0, 0x0),
    "errd5": (ERRD[2], 0, 0x0, 0x0),
}
# the sharded schedule needs bands taller than the halo: the layout tests' cases, and the tile case's chain
SHARD = {
    "cfg3-stream": (SHARD_CASES[0], 0, 0x3, 0x0),
    "tile": ((1, 150, 270, 100, 165, 4, u8, u8, 8, {}), 0, 0xC, 0x3),
    "rgb": (SHARD_CASES[2], 0, 0x0, 0x0),
}
# (sw, sh, nw, nh, channels, Tin, Tout, CLancIRParams fields, LANCIR kernels of a packed call)
LANCIR = {
    "c4-vector": (96, 54, 48, 27, 4, u8, u8, {}, ["lancir_col4_kernel", "lancir_row4_kernel"]),
    "c3-scalar": (77, 51, 47, 29, 3, f32, f32, {"kx": 1.3, "ky": 2.2}, ["lancir_col_kernel", "lancir_row_kernel"]),
}


def _is_errd(case):
    return case[0] >= 3 and np.dtype(case[7]).kind != "f"


def _no_f64(case):
    return np.dtype(case[6]) != np.float64 and np.dtype(case[7]) != np.float64 and not _is_errd(case)


def _lib():
    L = wlib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    L.avirb200_plan_kernel_paths.argtypes = [vp]
    L.avirb200_shard_workspace_bytes.argtypes = [vp, i, i, vp]
    L.lancirb200_resize_host.argtypes = [vp, vp, sz, vp, sz]
    L.lancirb200_plan_workspace_bytes.argtypes = [vp, vp]
    return L


def _rc(L, r, what):
    """The return code of a library call, with its message."""
    return r, (L.avirb200_last_error() or b"").decode() if r != 0 else "", what


def _assert_rc(res):
    r, msg, what = res
    assert r == 0, "%s returned %d: %s" % (what, r, msg)


@contextlib.contextmanager
def avir_case(name, table=AVIR, options=None):
    """A C-ABI plan of the named case with its kernel family, its kernel paths asserted."""
    case, family, must, never = table[name]
    with avir_plan(case, family, options) as (_, pl):
        L = _lib()
        paths = L.avirb200_plan_kernel_paths(pl)
        assert paths & must == must and paths & never == 0, (name, paths)
        yield L, pl, case


def _window_of(nw, nh, k=0):
    """An interior window at odd offsets (k: a different one per thread)."""
    w, h = max(1, nw // 2 - k), max(1, nh // 2 - (k % 3))
    x, y = min(nw - w, nw // 5 + 1 + k), min(nh - h, nh // 4 + 1 + k % 4)
    return (x, y, w, h)


# ---- one entry point on one plan, with its buffers ------------------------------------------------------------

class AvirCall:
    """An AVIR device entry point on one plan with its own device buffers; run(stream) enqueues it.

    entry: "device", "split" (row pass then column pass), "batch" (3 frames), "window" or "sharded"
    (avirb200_resize_sharded_local over `nranks` bands).  A window's footprint and workspace come from
    `sizer` (a plan of the same descriptor, so that the call's own plan is never queried) when given."""

    def __init__(self, L, pl, case, entry, win=None, nranks=0, sizer=None):
        import torch
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        self.L, self.pl, self.case, self.entry, self.win, self.nranks = L, pl, case, entry, win, nranks
        self.frames = 3 if entry == "batch" else 1
        self.ti, self.to = np.dtype(ti), np.dtype(to)
        self.frame_src = sh * sw * ch * self.ti.itemsize
        self.d_src = torch.empty(self.frames * self.frame_src, dtype=torch.uint8, device="cuda")
        if entry == "window":
            fi, n = WindowInfo(), C.c_size_t()
            qp = sizer if sizer is not None else pl
            _ok(L.avirb200_window_query(qp, *win, C.byref(fi)))
            _ok(L.avirb200_window_workspace_bytes(qp, *win, C.byref(n)))
            self.fi, nws = fi, n.value
            self.out_shape = (win[3], win[2], ch)
        else:
            self.out_shape = (nh, nw, ch)
            if entry == "sharded":
                nws = 0
                for r in range(nranks):
                    b = C.c_size_t()
                    _ok(L.avirb200_shard_workspace_bytes(pl, r, nranks, C.byref(b)))
                    nws += b.value
            else:
                b = C.c_size_t()
                _ok(L.avirb200_plan_workspace_bytes(pl, C.byref(b)))
                nws = b.value
        self.frame_dst = int(np.prod(self.out_shape)) * self.to.itemsize
        self.d_dst = torch.empty(self.frames * self.frame_dst, dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(max(nws, 1), dtype=torch.uint8, device="cuda")
        self.ws_bytes = nws
        self.src_pitch, self.dst_pitch = sw * ch, self.out_shape[1] * ch
        if entry == "batch":
            self.srcs = (C.c_void_p * 3)(*[self.d_src.data_ptr() + i * self.frame_src for i in range(3)])
            self.dsts = (C.c_void_p * 3)(*[self.d_dst.data_ptr() + i * self.frame_dst for i in range(3)])

    def source(self, seed):
        """The host bytes of the call's source for `seed` (batch: three frames)."""
        return np.concatenate([np.ascontiguousarray(cs.make_input(self.case, seed=seed + 1000 * i)).view(np.uint8)
                               .reshape(-1) for i in range(self.frames)])

    def poison(self):
        """Source poisoned, destination sentinel bytes, workspace 0xFF."""
        import torch
        p = np.full(self.d_src.numel() // self.ti.itemsize, cs.poison_of(self.ti), self.ti)
        self.d_src.copy_(torch.from_numpy(p.view(np.uint8)))
        self.d_dst.fill_(cs.SENTINEL)
        self.ws.fill_(0xFF)

    def run(self, st):
        L, pl = self.L, self.pl
        s, d, w = self.d_src.data_ptr(), self.d_dst.data_ptr(), self.ws.data_ptr()
        if self.entry == "device":
            return _rc(L, L.avirb200_resize_device(pl, s, self.src_pitch, d, self.dst_pitch, w, st), "resize_device")
        if self.entry == "split":
            r = _rc(L, L.avirb200_row_pass_device(pl, s, self.src_pitch, w, st), "row_pass_device")
            return r if r[0] else _rc(L, L.avirb200_col_pass_device(pl, w, d, self.dst_pitch, st), "col_pass_device")
        if self.entry == "batch":
            return _rc(L, L.avirb200_resize_device_batch(pl, 3, self.srcs, self.src_pitch, self.dsts, self.dst_pitch,
                                                         w, st), "resize_device_batch")
        if self.entry == "window":
            es = self.ti.itemsize
            sp = s + (self.fi.src_y0 * self.case[1] + self.fi.src_x0) * self.case[5] * es
            return _rc(L, L.avirb200_resize_window_device(pl, *self.win, sp, self.src_pitch, d, self.dst_pitch, w, st),
                       "resize_window_device")
        assert self.entry == "sharded"
        return _rc(L, L.avirb200_resize_sharded_local(pl, self.nranks, s, self.src_pitch, d, self.dst_pitch, w, st),
                   "resize_sharded_local")

    def out(self, buf=None):
        b = (self.d_dst if buf is None else buf).cpu().numpy()
        return b.view(self.to).reshape((self.frames,) + self.out_shape)

    def eager(self, src):
        """The call on the legacy stream, then a device synchronise: the reference."""
        import torch
        self.poison()
        self.d_src.copy_(torch.from_numpy(src))
        _assert_rc(self.run(None))
        torch.cuda.synchronize()
        return self.out()


class LancirCall:
    """A LANCIR device entry point ("device" or "window") on one plan with its own device buffers."""

    def __init__(self, L, pl, geom, entry, win=None):
        import torch
        sw, sh, nw, nh, ch, ti, to, kw = geom[:8]
        self.L, self.pl, self.geom, self.entry, self.win = L, pl, geom, entry, win
        self.frames = 1
        self.ti, self.to = np.dtype(ti), np.dtype(to)
        self.d_src = torch.empty(sh * sw * ch * self.ti.itemsize, dtype=torch.uint8, device="cuda")
        n = C.c_size_t()
        if entry == "window":
            fi = LancirWindowInfo()
            _ok(L.lancirb200_window_query(pl, *win, C.byref(fi)))
            _ok(L.lancirb200_window_workspace_bytes(pl, *win, C.byref(n)))
            self.fi = fi
            self.out_shape = (win[3], win[2], ch)
        else:
            _ok(L.lancirb200_plan_workspace_bytes(pl, C.byref(n)))
            self.out_shape = (nh, nw, ch)
        self.d_dst = torch.empty(int(np.prod(self.out_shape)) * self.to.itemsize, dtype=torch.uint8, device="cuda")
        self.ws = torch.empty(max(n.value, 1), dtype=torch.uint8, device="cuda")
        self.src_pitch, self.dst_pitch = sw * ch, self.out_shape[1] * ch

    def source(self, seed):
        sw, sh, nw, nh, ch, ti = self.geom[:6]
        return np.ascontiguousarray(o.lcg_image(sh, sw, ch, ti, seed=seed)).view(np.uint8).reshape(-1)

    poison = AvirCall.poison
    out = AvirCall.out
    eager = AvirCall.eager

    def run(self, st):
        L, pl = self.L, self.pl
        s, d, w = self.d_src.data_ptr(), self.d_dst.data_ptr(), self.ws.data_ptr()
        if self.entry == "device":
            return _rc(L, L.lancirb200_resize_device(pl, s, self.src_pitch, d, self.dst_pitch, w, st),
                       "lancirb200_resize_device")
        sp = s + (self.fi.src_y0 * self.geom[0] + self.fi.src_x0) * self.geom[4] * self.ti.itemsize
        return _rc(L, L.lancirb200_resize_window_device(pl, *self.win, sp, self.src_pitch, d, self.dst_pitch, w, st),
                   "lancirb200_resize_window_device")


@contextlib.contextmanager
def lancir_case(name):
    sw, sh, nw, nh, ch, ti, to, kw, _ = LANCIR[name]
    with lancir_plan(sw, sh, nw, nh, ch, ti, to, kw) as (_, pl, dp):
        L = _lib()
        llib()
        yield L, pl, LANCIR[name]


def _entries(case):
    out = ["device", "batch"]
    if _no_f64(case):
        out.insert(1, "split")
    if not _is_errd(case):
        out.append("window")
    return out


AVIR_ENTRY = [(n, e) for n in AVIR for e in _entries(AVIR[n][0])]
SHARD_ENTRY = [(n, k, ov) for n in SHARD for k in (2, 5) for ov in (3, 1)]
LANCIR_ENTRY = [(n, e) for n in LANCIR for e in ("device", "window")]


def _avir_call(L, pl, case, entry):
    fp, sw, sh, nw, nh = case[:5]
    return AvirCall(L, pl, case, entry, win=_window_of(nw, nh) if entry == "window" else None)


def _lancir_call(L, pl, geom, entry):
    return LancirCall(L, pl, geom, entry, win=_window_of(geom[2], geom[3]) if entry == "window" else None)


# ---- the anchor: one case per kernel family against upstream (or the C port) --------------------------------

@pytest.mark.parametrize("name", ["cfg3-stream", "tile", "tile-generic", "rgb", "f64", "errd4"])
def test_eager_reference_matches_upstream(name):
    with avir_case(name) as (L, pl, case):
        c = AvirCall(L, pl, case, "device")
        src = c.source(1)
        got = c.eager(src)[0]
        img = src.view(c.ti).reshape(case[2], case[1], case[5])
        assert cs.value_mismatch(expected(case, cs.source_layout(img)), got) == 0


@pytest.mark.skipif(not o.have_ref(), reason="needs oracle/_ref (upstream CLancIR)")
@pytest.mark.parametrize("name", list(LANCIR))
def test_lancir_eager_reference_matches_upstream(name):
    with lancir_case(name) as (L, pl, geom):
        sw, sh, nw, nh, ch, ti, to, kw, kernels = geom
        c = LancirCall(L, pl, geom, "device")
        src = c.source(1)
        got = c.eager(src)[0]
        r, want = o.lancir_ref(src.view(c.ti).reshape(sh, sw, ch), nw, nh, to, **kw)
        assert r == nh
        assert cs.value_mismatch(want, got) == 0


def lancir_route_failures():
    """(case, kernels launched, kernels named) of each LANCIR case whose packed call runs other kernels than
    it is named for; None when the profiler records no kernel activity."""
    import torch
    failures = []
    for name in LANCIR:
        with lancir_case(name) as (L, pl, geom):
            c = LancirCall(L, pl, geom, "device")
            c.eager(c.source(1))  # (kernels loaded)
            got = launched_kernels(lambda: _assert_rc(c.run(None)))
            if got is None:
                return None
            if got != geom[8]:
                failures.append((name, got, geom[8]))
    torch.cuda.synchronize()
    return failures


def test_lancir_cases_route_to_the_kernels_they_are_named_for():
    """Run in a child process: a profiler session leaves state behind in the process that runs it, and the
    other routing tests of the suite profile in this one."""
    code = ("import json, sys; sys.path[:0] = [%r, %r]; import test_gpu_streams as t; "
            "print(json.dumps(t.lancir_route_failures()))" % (ROOT, os.path.join(ROOT, "tests")))
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    failures = json.loads(r.stdout.strip().splitlines()[-1])
    if failures is None:
        pytest.skip("torch.profiler recorded no CUDA kernel activity on this machine")
    assert not failures, failures


# ---- 1. the caller's stream ------------------------------------------------------------------------------------

def on_side_stream(calls, seed=3):
    """Each call made eagerly first (the reference; it also loads the call's kernels, whose lazy loading
    may synchronise the context), then its buffers poisoned, then on one side stream S: a bounded spin,
    each call's real source, the calls in order, each destination copied out.  Asserts that S was still
    busy when the last call returned and that every copy equals its reference."""
    import torch
    hsrcs = [c.source(seed + i) for i, c in enumerate(calls)]
    refs = [c.eager(s) for c, s in zip(calls, hsrcs)]
    srcs = [torch.from_numpy(s).cuda() for s in hsrcs]
    for c in calls:
        c.poison()
    snaps = [torch.empty_like(c.d_dst) for c in calls]
    torch.cuda.synchronize()
    S = torch.cuda.Stream()
    with torch.cuda.stream(S):
        torch.cuda._sleep(SLEEP_CYCLES)
        results = []
        for c, s in zip(calls, srcs):
            c.d_src.copy_(s)
            results.append(c.run(S.cuda_stream))
        done = S.query()
        for c, snap in zip(calls, snaps):
            snap.copy_(c.d_dst)
    S.synchronize()
    for r in results:
        _assert_rc(r)
    assert not done, "the call waited for the caller's stream (S had finished when it returned)"
    for i, (c, snap) in enumerate(zip(calls, snaps)):
        assert cs.value_mismatch(refs[i], c.out(snap)) == 0, "call %d of %d" % (i + 1, len(calls))


@pytest.mark.parametrize("name,entry", AVIR_ENTRY)
def test_avir_call_runs_on_the_callers_stream(name, entry):
    with avir_case(name) as (L, pl, case):
        on_side_stream([_avir_call(L, pl, case, entry)])


@pytest.mark.parametrize("name,nranks,overlap", SHARD_ENTRY)
def test_sharded_local_runs_on_the_callers_stream(name, nranks, overlap):
    with avir_case(name, SHARD, {ab.OPT_OVERLAP_HALO: overlap}) as (L, pl, case):
        on_side_stream([AvirCall(L, pl, case, "sharded", nranks=nranks)])


@pytest.mark.parametrize("name,entry", LANCIR_ENTRY)
def test_lancir_call_runs_on_the_callers_stream(name, entry):
    with lancir_case(name) as (L, pl, geom):
        on_side_stream([_lancir_call(L, pl, geom, entry)])


def test_two_plans_back_to_back_share_one_workspace():
    """Two plans' calls queued on one stream with no synchronise between them, one workspace: the stream
    alone keeps the second call's passes behind the first's."""
    import torch
    with avir_case("cfg3-stream") as (L, pa, ca), avir_case("tile") as (_, pb, cb):
        a, b = AvirCall(L, pa, ca, "device"), AvirCall(L, pb, cb, "device")
        ws = torch.empty(max(a.ws.numel(), b.ws.numel()), dtype=torch.uint8, device="cuda")
        a.ws = b.ws = ws
        on_side_stream([a, b])


# ---- 2. graph capture ------------------------------------------------------------------------------------------

def capture_and_replay(c, warm_up=True, replays=3, ref_call=None):
    """Captures c.run on a side stream (global capture mode) and replays it over new sources; each replay
    must equal the eager call (of ref_call when given, else of c itself) on the same source."""
    import torch
    srcs = [c.source(20 + i) for i in range(replays + 1)]
    refs = [(ref_call or c).eager(s) for s in srcs]
    d_srcs = [torch.from_numpy(s).cuda() for s in srcs]
    c.poison()
    torch.cuda.synchronize()
    S = torch.cuda.Stream()
    if warm_up:
        with torch.cuda.stream(S):
            c.d_src.copy_(d_srcs[0])
            _assert_rc(c.run(S.cuda_stream))
        S.synchronize()
    g = torch.cuda.CUDAGraph()
    res, err = None, None
    try:
        with torch.cuda.graph(g, stream=S):
            res = c.run(S.cuda_stream)
    except RuntimeError as e:  # the capture was invalidated: report the library's own account first
        err = e
    assert res is not None, err
    _assert_rc(res)
    assert err is None, err
    for i in range(1, replays + 1):
        c.d_src.copy_(d_srcs[i])
        c.d_dst.fill_(cs.SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        assert cs.value_mismatch(refs[i], c.out()) == 0, "replay %d" % i
    del g


@pytest.mark.parametrize("name,entry", AVIR_ENTRY)
def test_avir_call_in_a_cuda_graph(name, entry):
    with avir_case(name) as (L, pl, case):
        capture_and_replay(_avir_call(L, pl, case, entry))


@pytest.mark.parametrize("name,nranks,overlap", SHARD_ENTRY)
def test_sharded_local_in_a_cuda_graph(name, nranks, overlap):
    """The fused schedule's mailbox comes from cudaMallocAsync on the caller's stream: a graph memory node."""
    with avir_case(name, SHARD, {ab.OPT_OVERLAP_HALO: overlap}) as (L, pl, case):
        capture_and_replay(AvirCall(L, pl, case, "sharded", nranks=nranks))


@pytest.mark.parametrize("name,entry", LANCIR_ENTRY)
def test_lancir_call_in_a_cuda_graph(name, entry):
    with lancir_case(name) as (L, pl, geom):
        capture_and_replay(_lancir_call(L, pl, geom, entry))


def test_unqueried_window_first_called_inside_a_capture():
    """A window the plan was never asked about (its footprint and workspace from a twin plan of the same
    descriptor), whose first call is captured: the launch must not build the tile kernel's range tables
    (an allocation and a synchronous copy), and its pixels are the queried window's."""
    import torch
    with avir_case("tile") as (L, pl, case), avir_case("tile") as (_, twin, _c):
        fp, sw, sh, nw, nh = case[:5]
        win = _window_of(nw, nh, 5)
        queried = AvirCall(L, twin, case, "window", win=win)
        c = AvirCall(L, pl, case, "window", win=win, sizer=twin)
        # the kernels of both families loaded (module loading is not what this test is about), through
        # calls that build no table of this window on `pl`; the references come from the twin
        src = c.source(40)
        AvirCall(L, pl, case, "device").eager(src)
        with avir_case("tile-generic") as (_, gen, _c2):
            AvirCall(L, gen, case, "device").eager(src)
        torch.cuda.synchronize()
        capture_and_replay(c, warm_up=False, ref_call=queried)
        assert cs.value_mismatch(queried.eager(src), c.eager(src)) == 0


# ---- 3. threads ------------------------------------------------------------------------------------------------

def run_threads(n, body):
    """body(i) in n threads; re-raises the first failure after every thread has been joined."""
    errors = []

    def wrap(i):
        try:
            body(i)
        except BaseException as e:  # noqa: BLE001
            errors.append((i, e))

    ts = [threading.Thread(target=wrap, args=(i,)) for i in range(n)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    if errors:
        i, e = errors[0]
        raise AssertionError("thread %d of %d failed: %r" % (i, n, e)) from e


def thread_calls(make, refs, srcs):
    """THREADS threads, each with its own call (make(i): own buffers and workspace) and stream, making
    CALLS_PER_THREAD calls over the seeded sources; refs[seed](i) is what thread i must get."""
    import torch

    def body(i):
        c = make(i)
        s = torch.cuda.Stream()
        for k in range(CALLS_PER_THREAD):
            seed = (i + k) % len(srcs)
            with torch.cuda.stream(s):
                c.d_src.copy_(srcs[seed])
                c.d_dst.fill_(cs.SENTINEL)
                res = c.run(s.cuda_stream)
            s.synchronize()
            _assert_rc(res)
            assert cs.value_mismatch(refs[seed](i), c.out()) == 0, ("seed", seed)

    run_threads(THREADS, body)


@pytest.mark.parametrize("entry", ["device", "window"])
@pytest.mark.parametrize("name", ["cfg3-stream", "tile", "tile-generic", "rgb", "f64"])
def test_avir_threads_share_a_plan(name, entry):
    """8 threads on one plan; window threads each query their own window inside the thread (the plan's
    range tables are built concurrently)."""
    import torch
    with avir_case(name) as (L, pl, case):
        fp, sw, sh, nw, nh = case[:5]
        full = AvirCall(L, pl, case, "device")
        hsrcs = [full.source(50 + k) for k in range(THREADS)]
        fulls = [full.eager(s)[0] for s in hsrcs]
        srcs = [torch.from_numpy(s).cuda() for s in hsrcs]
        wins = [_window_of(nw, nh, i) for i in range(THREADS)]
        if entry == "device":
            refs = [(lambda i, f=f: f[None]) for f in fulls]
            thread_calls(lambda i: AvirCall(L, pl, case, "device"), refs, srcs)
        else:
            refs = [(lambda i, f=f: crop(f, wins[i])[None]) for f in fulls]
            thread_calls(lambda i: AvirCall(L, pl, case, "window", win=wins[i]), refs, srcs)


@pytest.mark.parametrize("name", list(LANCIR))
def test_lancir_threads_share_a_plan(name):
    import torch
    with lancir_case(name) as (L, pl, geom):
        full = LancirCall(L, pl, geom, "device")
        hsrcs = [full.source(50 + k) for k in range(THREADS)]
        refs = [(lambda i, f=full.eager(s): f) for s in hsrcs]
        srcs = [torch.from_numpy(s).cuda() for s in hsrcs]
        thread_calls(lambda i: LancirCall(L, pl, geom, "device"), refs, srcs)


HOST_THREADS = 4


def _host_buffers(n_src, n_dst, src_dtype, dst_dtype, pinned):
    return cs.host_array(n_src, src_dtype, pinned), cs.host_array(n_dst, dst_dtype, pinned)


@pytest.mark.parametrize("bands", [1, 3])
@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("plans", ["shared", "several"])
@pytest.mark.parametrize("name", ["cfg3-stream", "tile"])
def test_avir_host_threads(name, plans, pinned, bands):
    """avirb200_resize_host from several threads, on one plan (the plan's mutex) or one plan per thread on
    the same device (the device's staging mutex), unbanded and in 3 row bands."""
    case = AVIR[name][0]
    fp, sw, sh, nw, nh, ch, ti, to = case[:8]
    with contextlib.ExitStack() as stack:
        nplans = 1 if plans == "shared" else HOST_THREADS
        pls = [stack.enter_context(avir_case(name, options={ab.OPT_HOST_BANDS: bands}))[1] for _ in range(nplans)]
        L = _lib()
        full = AvirCall(L, pls[0], case, "device")
        hsrcs = [full.source(60 + k) for k in range(HOST_THREADS)]
        refs = [full.eager(s)[0] for s in hsrcs]

        def body(i):
            pl = pls[i % nplans]
            h_src, h_dst = _host_buffers(sh * sw * ch, nh * nw * ch, ti, to, pinned)
            for k in range(2):
                seed = (i + k) % HOST_THREADS
                h_src[:] = hsrcs[seed].view(ti)
                h_dst.view(np.uint8)[:] = cs.SENTINEL
                _assert_rc(_rc(L, L.avirb200_resize_host(pl, h_src.ctypes.data, sw * ch, h_dst.ctypes.data, nw * ch),
                               "resize_host"))
                assert cs.value_mismatch(refs[seed], h_dst.reshape(nh, nw, ch)) == 0, ("seed", seed)

        run_threads(HOST_THREADS, body)


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("name", ["cfg3-stream", "tile"])
def test_avir_window_host_threads(name, pinned):
    case = AVIR[name][0]
    fp, sw, sh, nw, nh, ch, ti, to = case[:8]
    with avir_case(name) as (L, pl, _):
        full = AvirCall(L, pl, case, "device")
        hsrcs = [full.source(70 + k) for k in range(HOST_THREADS)]
        refs = [full.eager(s)[0] for s in hsrcs]

        def body(i):
            win = _window_of(nw, nh, i)
            h_src, h_dst = _host_buffers(sh * sw * ch, win[2] * win[3] * ch, ti, to, pinned)
            for k in range(2):
                seed = (i + k) % HOST_THREADS
                h_src[:] = hsrcs[seed].view(ti)
                _assert_rc(_rc(L, L.avirb200_resize_window_host(pl, *win, h_src.ctypes.data, sw * ch, h_dst.ctypes.data,
                                                                win[2] * ch), "resize_window_host"))
                assert cs.value_mismatch(crop(refs[seed], win), h_dst.reshape(win[3], win[2], ch)) == 0, ("seed", seed)

        run_threads(HOST_THREADS, body)


@pytest.mark.parametrize("pinned", [False, True], ids=["pageable", "pinned"])
@pytest.mark.parametrize("name", list(LANCIR))
def test_lancir_host_threads(name, pinned):
    """lancirb200_resize_host and lancirb200_resize_window_host from several threads on one plan."""
    with lancir_case(name) as (L, pl, geom):
        sw, sh, nw, nh, ch, ti, to = geom[:7]
        full = LancirCall(L, pl, geom, "device")
        hsrcs = [full.source(80 + k) for k in range(HOST_THREADS)]
        refs = [full.eager(s)[0] for s in hsrcs]

        def body(i):
            win = _window_of(nw, nh, i)
            h_src, h_dst = _host_buffers(sh * sw * ch, nh * nw * ch, ti, to, pinned)
            for k in range(2):
                seed = (i + k) % HOST_THREADS
                h_src[:] = hsrcs[seed].view(ti)
                _assert_rc(_rc(L, L.lancirb200_resize_host(pl, h_src.ctypes.data, sw * ch, h_dst.ctypes.data, nw * ch),
                               "lancirb200_resize_host"))
                assert cs.value_mismatch(refs[seed], h_dst.reshape(nh, nw, ch)) == 0, ("seed", seed)
                _assert_rc(_rc(L, L.lancirb200_resize_window_host(pl, *win, h_src.ctypes.data, sw * ch,
                                                                  h_dst.ctypes.data, win[2] * ch),
                               "lancirb200_resize_window_host"))
                got = h_dst[:win[2] * win[3] * ch].reshape(win[3], win[2], ch)
                assert cs.value_mismatch(crop(refs[seed], win), got) == 0, ("window seed", seed)

        run_threads(HOST_THREADS, body)


# ---- host calls leave the caller's current device alone ---------------------------------------------------------

def test_host_calls_restore_the_callers_device():
    """A plan on device 1 called from a thread whose current device is 0: the call runs on the plan's
    device and device 0 is current again afterwards (read through the driver, not through torch)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    cuda = C.CDLL("libcuda.so.1")

    def current():
        d = C.c_int(-1)
        assert cuda.cuCtxGetDevice(C.byref(d)) == 0
        return d.value

    geom = LANCIR["c4-vector"]
    sw, sh, nw, nh, ch, ti, to, kw = geom[:8]
    src = o.lcg_image(sh, sw, ch, ti, seed=90)
    win = _window_of(nw, nh)
    outs = {}
    for dev in (0, 1):
        torch.cuda.set_device(dev)
        with lancir_plan(sw, sh, nw, nh, ch, ti, to, kw) as (L, pl, _):
            _lib()
            torch.cuda.set_device(0)
            assert current() == 0
            full = np.zeros((nh, nw, ch), to)
            part = np.zeros((win[3], win[2], ch), to)
            _ok(L.lancirb200_resize_host(pl, src.ctypes.data, sw * ch, full.ctypes.data, nw * ch))
            assert current() == 0, "lancirb200_resize_host left device %d current" % current()
            _ok(L.lancirb200_resize_window_host(pl, *win, src.ctypes.data, sw * ch, part.ctypes.data, win[2] * ch))
            assert current() == 0, "lancirb200_resize_window_host left device %d current" % current()
            outs[dev] = (full, part)
            torch.cuda.set_device(dev)  # (the plan is destroyed on its own device)
    torch.cuda.set_device(0)
    assert cs.value_mismatch(outs[0][0], outs[1][0]) == 0
    assert cs.value_mismatch(crop(outs[0][0], win), outs[1][1]) == 0

    # AVIR's three host calls (the sharded one as its single rank)
    case = AVIR["tile"][0]
    fp, sw, sh, nw, nh, ch, ti, to = case[:8]
    src = cs.make_input(case, seed=91)
    win = _window_of(nw, nh)
    outs = {}
    for dev in (0, 1):
        torch.cuda.set_device(dev)
        with avir_case("tile") as (L, pl, _):
            L.avirb200_resize_sharded_host.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                       C.c_size_t, C.c_void_p, C.c_size_t]
            torch.cuda.set_device(0)
            assert current() == 0
            full, band = np.zeros((nh, nw, ch), to), np.zeros((nh, nw, ch), to)
            part = np.zeros((win[3], win[2], ch), to)
            _ok(L.avirb200_resize_host(pl, src.ctypes.data, sw * ch, full.ctypes.data, nw * ch))
            assert current() == 0, "avirb200_resize_host left device %d current" % current()
            _ok(L.avirb200_resize_window_host(pl, *win, src.ctypes.data, sw * ch, part.ctypes.data, win[2] * ch))
            assert current() == 0, "avirb200_resize_window_host left device %d current" % current()
            _ok(L.avirb200_resize_sharded_host(pl, None, 0, 1, src.ctypes.data, sw * ch, band.ctypes.data, nw * ch))
            assert current() == 0, "avirb200_resize_sharded_host left device %d current" % current()
            outs[dev] = (full, part, band)
            torch.cuda.set_device(dev)  # (the plan is destroyed on its own device)
    torch.cuda.set_device(0)
    assert cs.value_mismatch(outs[0][0], outs[1][0]) == 0
    assert cs.value_mismatch(crop(outs[0][0], win), outs[1][1]) == 0
    assert cs.value_mismatch(outs[0][0], outs[1][2]) == 0
