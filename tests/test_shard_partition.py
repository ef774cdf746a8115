"""The band partition both resizers' row-sharded calls share, and the sizes derived from it.

Rank r of n holds source rows [src_h r / n, src_h (r + 1) / n) and produces destination rows
[dst_h r / n, dst_h (r + 1) / n); a rank left without rows is refused.  AVIR and CLancIR differ only in which
rows a band reads (AVIR: intermediate rows of its column chain; CLancIR: source rows of its vertical
footprint), so on the same heights both must report the same four split fields and refuse the same empty
bands.  Heights cover one-row bands, uneven splits and images past 65535 rows, at 1 to 9 ranks.  The workspace
and mailbox sizes are checked against the arithmetic the library documents."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
from test_lancir_sharding import ShardInfo
from test_lancir_window import Descriptor
from test_sharded_errd import _a256, mailbox_bytes, shard_workspace_bytes

ERR_UNSUPPORTED = -4
SRC_W, DST_W, CH = 4, 2, 4
RANKS = range(1, 10)
# (source rows, destination rows)
HEIGHTS = [(1, 1), (2, 1), (1, 3), (9, 9), (9, 2), (10, 7), (37, 101), (101, 37), (1000, 999), (70001, 35000),
           (35000, 70001), (65536, 65537)]
FIELDS = ("src_row0", "src_rows", "dst_row0", "dst_rows")


def split(rows, rank, nranks):
    r0 = rows * rank // nranks
    return r0, rows * (rank + 1) // nranks - r0


def avir_case(sh, nh):
    return (1, SRC_W, sh, DST_W, nh, CH, np.float32, np.float32, 16, {})


def lancir_case(sh, nh):
    return (SRC_W, sh, DST_W, nh, CH, np.float32, np.float32, {})


class AvirDescriptor:
    def __init__(self, sh, nh):
        case = avir_case(sh, nh)
        rs, v = cs.resizer_and_vars(case)
        self.handle, self.ptr, _ = rs.descriptor((sh, SRC_W, CH), np.float32, DST_W, nh, np.float32, 0.0, v)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        ab.CImageResizer.free_descriptor(self.handle)


def query(fn, dp, rank, nranks):
    si = ShardInfo()
    rc = fn(C.c_void_p(dp), rank, nranks, C.byref(si))
    return rc, si, ab.lib().avirb200_last_error().decode() if rc != 0 else ""


def fields(si):
    return tuple(getattr(si, f) for f in FIELDS)


@pytest.mark.parametrize("sh,nh", HEIGHTS, ids=lambda v: str(v))
def test_both_resizers_split_alike(sh, nh):
    L = ab.lib()
    with AvirDescriptor(sh, nh) as ad, Descriptor(lancir_case(sh, nh)) as ld:
        for n in RANKS:
            for r in range(n):
                want = split(sh, r, n) + split(nh, r, n)
                ra, a, ma = query(L.avirb200_shard_query_desc, ad.ptr, r, n)
                rl, l, ml = query(L.lancirb200_shard_query_desc, ld.ptr, r, n)
                if want[1] <= 0 or want[3] <= 0:
                    assert ra == rl == ERR_UNSUPPORTED, (r, n, ra, rl)
                    assert ma == ml == "image has fewer rows than ranks", (r, n)
                    continue
                assert fields(a) == fields(l) == want, (r, n)
                for rc, si, msg in ((ra, a, ma), (rl, l, ml)):
                    if rc != 0:
                        assert rc == ERR_UNSUPPORTED, (r, n, rc)
                        assert msg in ("halo exceeds the neighbouring band (too many ranks)",
                                       "band too tall (more than 65535 destination rows)"), (r, n, msg)
                        continue
                    assert si.need_row0 == si.src_row0 - si.halo_up and si.halo_up >= 0 and si.halo_down >= 0
                    assert si.need_rows == si.halo_up + si.src_rows + si.halo_down
                    if r > 0:
                        assert si.halo_up <= split(sh, r - 1, n)[1], (r, n)
                    if r + 1 < n:
                        assert si.halo_down <= split(sh, r + 1, n)[1], (r, n)
                # (CLancIR's kernels take at most 65535 destination rows per band)
                assert (ml == "band too tall (more than 65535 destination rows)") == (want[3] > 65535), (r, n)


@pytest.mark.parametrize("sh,nh", HEIGHTS, ids=lambda v: str(v))
def test_avir_shard_layout_matches_its_arithmetic(sh, nh):
    L = ab.lib()
    L.avirb200_shard_layout_desc.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    with AvirDescriptor(sh, nh) as ad:
        for n in RANKS:
            for r in range(n):
                rq, si, _ = query(L.avirb200_shard_query_desc, ad.ptr, r, n)
                ws, box = C.c_size_t(), C.c_size_t()
                rc = L.avirb200_shard_layout_desc(C.c_void_p(ad.ptr), r, n, C.byref(ws), C.byref(box))
                assert rc == rq, (r, n)
                if rc != 0:
                    continue
                info = {k: getattr(si, k) for k, _ in si._fields_}
                assert ws.value == shard_workspace_bytes(info, SRC_W, DST_W, CH, False, False, False), (r, n)
                assert box.value == mailbox_bytes(info, DST_W, CH, False, 2), (r, n)


def lancir_shard_workspace_bytes(si):
    """The band's intermediate (dst_rows x src_w x channels floats), its two halo segments (rows of src_w x
    channels elements, 16-byte aligned) and the 256-byte header of the flags, each 256-byte aligned."""
    row16 = (SRC_W * CH * 4 + 15) // 16 * 16
    return _a256(si.dst_rows * SRC_W * CH * 4) + _a256(si.halo_up * row16) + _a256(si.halo_down * row16) + 256


@pytest.mark.gpu
@pytest.mark.parametrize("sh,nh", HEIGHTS, ids=lambda v: str(v))
def test_lancir_shard_workspace_matches_its_arithmetic(sh, nh):
    L = ab.lib()
    vp, i = C.c_void_p, C.c_int
    L.lancirb200_plan_create.argtypes = [vp, vp]
    L.lancirb200_plan_destroy.argtypes = [vp]
    L.lancirb200_shard_workspace_bytes.argtypes = [vp, i, i, vp]
    with Descriptor(lancir_case(sh, nh)) as ld:
        pl = C.c_void_p()
        assert L.lancirb200_plan_create(C.c_void_p(ld.ptr), C.byref(pl)) == 0, L.avirb200_last_error()
        try:
            for n in RANKS:
                for r in range(n):
                    rq, si, _ = query(L.lancirb200_shard_query_desc, ld.ptr, r, n)
                    b = C.c_size_t()
                    rc = L.lancirb200_shard_workspace_bytes(pl, r, n, C.byref(b))
                    assert rc == rq, (r, n)
                    if rc == 0:
                        assert b.value == lancir_shard_workspace_bytes(si), (r, n)
        finally:
            L.lancirb200_plan_destroy(pl)
