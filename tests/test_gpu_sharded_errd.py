"""Double buffers and error diffusion on the sharded and per-pass entry points (run with -m gpu on an H100).

Every band of avirb200_resize_sharded_local must equal the same rows of avirb200_resize_device and upstream
(or the C port): 0 mismatching elements.  Error diffusion hands each band's last D row to the next band
through the band's mailbox; double buffers are cast per band.  The multi-GPU form runs in
sharded_errd_worker.py, one process per GPU, and needs at least two GPUs."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
from test_gpu_layouts import (_ok, avir_plan, dptr, expected, guarded_workspace, make_layouts, plan_workspace,
                              tail_damage, to_device)
from test_sharded_errd import mailbox_bytes, shard_layout, shard_workspace_bytes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
FAMILIES = pytest.mark.parametrize("family", [0, 2, 1], ids=["product", "tile", "generic"])

ERRD = [
    (3, 160, 216, 80, 108, 4, u8, u8, 8, {}),
    (4, 160, 216, 80, 108, 3, u8, u8, 8, {}),
    (5, 160, 216, 80, 108, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),  # cfg5's class and epilogue
    (5, 160, 216, 80, 108, 2, u16, u16, 16, {}),
    (4, 160, 216, 80, 108, 1, u16, u16, 16, {}),
    (3, 160, 216, 80, 108, 4, u8, u8, 6, {"gamma": True, "alpha": 0}),  # bit-depth truncation
]
F64 = [
    (1, 192, 216, 96, 108, 4, f64, f64, 16, {}),
    (2, 192, 216, 96, 108, 3, f64, u8, 8, {}),
    (1, 192, 216, 96, 108, 4, u8, f64, 8, {"gamma": True, "alpha": 3}),
    (5, 192, 216, 96, 108, 4, f64, u8, 8, {}),  # double source, dithered output
]


def _lib(L):
    vp = C.c_void_p
    L.avirb200_shard_workspace_bytes.argtypes = [vp, C.c_int, C.c_int, vp]
    return L


def shard_ws(L, pl, nranks):
    sizes = []
    for r in range(nranks):
        b = C.c_size_t()
        _ok(L.avirb200_shard_workspace_bytes(pl, r, nranks, C.byref(b)))
        sizes.append(b.value)
    return sizes


def device_result(L, pl, case, sl):
    """avirb200_resize_device on the same source: the reference of every band."""
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    d_src = to_device(sl)
    out = torch.empty(nh * nw * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
    ws = torch.empty(plan_workspace(L, pl), dtype=torch.uint8, device="cuda")
    _ok(L.avirb200_resize_device(pl, dptr(d_src, sl), sl.pitch, out.data_ptr(), nw * ch, ws.data_ptr(), None))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(to).reshape(nh, nw, ch)


def run_sharded_local(L, pl, case, sl, dl, nranks):
    """The sharded call over guarded buffers and a workspace of exactly the shards' bytes with a sentinel tail:
    (destination image, bytes stored past the workspace)."""
    import torch
    n = sum(shard_ws(L, pl, nranks))
    d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
    ws[:n].fill_(0xFF)
    _ok(L.avirb200_resize_sharded_local(pl, nranks, dptr(d_src, sl), sl.pitch, dptr(d_dst, dl), dl.pitch,
                                        ws.data_ptr(), None))
    torch.cuda.synchronize()
    back = d_dst.cpu().numpy().view(dl.backing.dtype)
    assert cs.guard_damage(dl, back) == 0, "destination guard bytes overwritten"
    assert np.array_equal(d_src.cpu().numpy(), sl.backing.view(np.uint8)), "source buffer written"
    return np.ascontiguousarray(dl.view(back)), tail_damage(ws, n)


def check_sharded(case, nranks, overlap, family, layout="L0-packed", src=None):
    sl, dl = make_layouts(case, layout, seed=5)
    if src is not None:
        sl = cs.source_layout(src, sl.pitch - case[1] * case[5])
    with avir_plan(case, family, {ab.OPT_OVERLAP_HALO: overlap}) as (L, pl):
        L = _lib(L)
        want = device_result(L, pl, case, sl)
        got, tail = run_sharded_local(L, pl, case, sl, dl, nranks)
        assert cs.value_mismatch(want, got) == 0, "sharded_local != resize_device"
        assert tail == 0, "store past the shards' workspace"
    return sl, got


@FAMILIES
@pytest.mark.parametrize("overlap", [3, 1])
@pytest.mark.parametrize("nranks", [2, 3, 5, 8])
@pytest.mark.parametrize("case", ERRD, ids=cs.case_id)
def test_sharded_local_errd_matches_device_and_upstream(case, nranks, overlap, family):
    sl, got = check_sharded(case, nranks, overlap, family)
    assert cs.value_mismatch(expected(case, sl), got) == 0, "sharded_local != upstream"


@FAMILIES
@pytest.mark.parametrize("overlap", [3, 1])
@pytest.mark.parametrize("nranks", [2, 5])
@pytest.mark.parametrize("case", F64, ids=cs.case_id)
def test_sharded_local_double_matches_device_and_upstream(case, nranks, overlap, family):
    sl, got = check_sharded(case, nranks, overlap, family)
    assert cs.value_mismatch(expected(case, sl), got) == 0, "sharded_local != upstream"


@pytest.mark.parametrize("kind", ["range", "huge", "nonfinite", "tiny"])
@pytest.mark.parametrize("case", [F64[0], F64[1], F64[3]], ids=cs.case_id)
def test_sharded_local_double_value_domain(case, kind):
    """Sources beyond float's range (+-1e39, 1e300), double subnormals, NaN positions."""
    check_sharded(case, 3, 3, 0, src=cs.value_image(case, kind))


@pytest.mark.parametrize("layout", ["L1-src-pad4", "L3-src-offset1", "L4-dst-pad2", "L5-dst-odd"])
@pytest.mark.parametrize("case", [ERRD[2], ERRD[3], F64[0], F64[1]], ids=cs.case_id)
def test_sharded_local_layouts(case, layout):
    """Padded and offset band buffers with poisoned source padding and destination sentinels."""
    check_sharded(case, 3, 3, 0, layout=layout)


@FAMILIES
@pytest.mark.parametrize("case", ERRD + F64, ids=cs.case_id)
def test_split_passes_match_resize_device(case, family):
    """avirb200_row_pass_device then avirb200_col_pass_device = avirb200_resize_device = upstream."""
    import torch
    for layout in ("L0-packed", "L6-src-pad4-dst-odd"):
        sl, dl = make_layouts(case, layout, seed=4)
        with avir_plan(case, family) as (L, pl):
            n = plan_workspace(L, pl)
            d_src, d_dst, ws = to_device(sl), to_device(dl), guarded_workspace(n)
            _ok(L.avirb200_row_pass_device(pl, dptr(d_src, sl), sl.pitch, ws.data_ptr(), None))
            _ok(L.avirb200_col_pass_device(pl, ws.data_ptr(), dptr(d_dst, dl), dl.pitch, None))
            torch.cuda.synchronize()
            back = d_dst.cpu().numpy().view(dl.backing.dtype)
            got = np.ascontiguousarray(dl.view(back))
            assert cs.value_mismatch(device_result(L, pl, case, sl), got) == 0, layout
            assert cs.value_mismatch(expected(case, sl), got) == 0, layout
            assert cs.guard_damage(dl, back) == 0
            assert tail_damage(ws, n) == 0


@pytest.mark.parametrize("case", ERRD + F64, ids=cs.case_id)
def test_shard_workspace_matches_layout_query(case):
    """avirb200_shard_workspace_bytes of a created plan is what avirb200_shard_layout_desc computes from the
    descriptor and the restated ws_layout arithmetic; the mailbox bytes are MailboxLayout's, restated."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    errd = fp >= 3 and np.dtype(to).kind != "f"
    with avir_plan(case) as (L, pl):
        L = _lib(L)
        for nranks in (2, 5, 8):
            sizes = shard_ws(L, pl, nranks)
            for r in range(nranks):
                code, ws, box, si = shard_layout(case, r, nranks)
                assert code == 0
                assert sizes[r] == ws == shard_workspace_bytes(si, sw, nw, ch, np.dtype(ti) == f64,
                                                               np.dtype(to) == f64, errd), (nranks, r)
                assert box == mailbox_bytes(si, nw, ch, errd, 2), (nranks, r)


@pytest.mark.parametrize("case", [ERRD[0], F64[0], F64[2]], ids=cs.case_id)
def test_sharded_destination_pitch_smaller_than_a_row_is_refused(case):
    """Double output and error diffusion write the caller's rows at its pitch after the column pass: a pitch
    below a row is AVIRB200_ERR_BAD_ARG, as on avirb200_resize_device, before any launch."""
    import torch
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    with avir_plan(case) as (L, pl):
        L = _lib(L)
        L.avirb200_resize_sharded.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                              C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        buf = torch.zeros(1 << 24, dtype=torch.uint8, device="cuda")
        p = buf.data_ptr()
        assert L.avirb200_resize_sharded_local(pl, 2, p, sw * ch, p, nw * ch - 1, p, None) == -1
        assert L.avirb200_resize_sharded(pl, None, 0, 1, p, sw * ch, p, nw * ch - 1, p, None) == -1
        torch.cuda.synchronize()


def test_consecutive_calls_with_different_inputs():
    """Three and more calls on one plan and one workspace, new sources each time (the mailbox slots of
    consecutive calls)."""
    import torch
    for case in (ERRD[2], F64[3]):
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
        with avir_plan(case) as (L, pl):
            L = _lib(L)
            n = sum(shard_ws(L, pl, 5))
            ws = torch.empty(n, dtype=torch.uint8, device="cuda")
            d_dst = torch.empty(nh * nw * ch * np.dtype(to).itemsize, dtype=torch.uint8, device="cuda")
            for seed in range(4):
                src = cs.make_input(case, seed=40 + seed)
                sl = cs.source_layout(src)
                d_src = to_device(sl)
                _ok(L.avirb200_resize_sharded_local(pl, 5, dptr(d_src, sl), sl.pitch, d_dst.data_ptr(), nw * ch,
                                                    ws.data_ptr(), None))
                torch.cuda.synchronize()
                got = d_dst.cpu().numpy().view(to).reshape(nh, nw, ch)
                assert cs.value_mismatch(device_result(L, pl, case, sl), got) == 0, seed


FULL = {
    "cfg5-errd": (5, 7680, 4320, 1920, 1080, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),
    "16k-u16-errd": (4, 16384, 16384, 4096, 4096, 4, u16, u16, 16, {}),
}


@pytest.mark.parametrize("name", list(FULL))
def test_full_size_errd_over_8_bands(name):
    import torch
    case = FULL[name]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    TT = {u8: torch.uint8, u16: torch.uint16}
    g = torch.Generator(device="cuda").manual_seed(9)
    src = torch.randint(0, np.iinfo(ti).max + 1, (sh, sw, ch), generator=g, device="cuda", dtype=torch.int32).to(TT[ti])
    with avir_plan(case) as (L, pl):
        L = _lib(L)
        ws = torch.empty(max(plan_workspace(L, pl), sum(shard_ws(L, pl, 8))), dtype=torch.uint8, device="cuda")
        a = torch.empty((nh, nw, ch), dtype=TT[to], device="cuda")
        b = torch.full((nh, nw, ch), 7, dtype=TT[to], device="cuda")
        _ok(L.avirb200_resize_device(pl, src.data_ptr(), sw * ch, a.data_ptr(), nw * ch, ws.data_ptr(), None))
        torch.cuda.synchronize()
        _ok(L.avirb200_resize_sharded_local(pl, 8, src.data_ptr(), sw * ch, b.data_ptr(), nw * ch, ws.data_ptr(), None))
        torch.cuda.synchronize()
        assert int((a.view(torch.uint8) != b.view(torch.uint8)).sum().item()) == 0


def _gpus():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


@pytest.mark.parametrize("nranks", [2, 4, 8])
def test_multi_gpu_sharded_errd_and_double(nranks):
    """avirb200_resize_sharded, one process per GPU, fused (3), push (1) and NCCL (0) schedules."""
    if _gpus() < nranks:
        pytest.skip("needs %d GPUs" % nranks)
    port = 29700 + (os.getpid() % 200) + nranks
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nranks),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "sharded_errd_worker.py")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    print(r.stdout[-4000:])
    assert r.returncode == 0, r.stdout[-4000:]
    assert "mismatches=" in r.stdout
