"""Row-sharded CLancIR without a GPU: the bands lancirb200_shard_query_desc reports.

Rank r of n holds source rows [src_h r / n, src_h (r + 1) / n) and produces destination rows
[dst_h r / n, dst_h (r + 1) / n).  Its `need` rows are SOURCE rows: the band's vertical footprint (every tap
position of its destination rows, clamped to the image) joined with its own source band; the halos are the
rows of it its neighbours hold.  Checked: the partition's consistency, `need` against brute force, and on the
oracle's C port that a source poisoned outside a band's `need` rows still gives that band's destination rows
the whole image's bits."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import oracle_ref as o
from test_lancir_window import CASES, Descriptor, _poisons, brute_span, case_id, port_resize

ERR_BAD_ARG, ERR_UNSUPPORTED = -1, -4
RANKS = (2, 3, 5, 8)


class ShardInfo(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_row0", "src_rows", "dst_row0", "dst_rows", "need_row0", "need_rows",
                                         "halo_up", "halo_down")]


def shard_query_desc(dp, rank, nranks):
    si = ShardInfo()
    rc = ab.lib().lancirb200_shard_query_desc(C.c_void_p(dp), rank, nranks, C.byref(si))
    return rc, si


def bands(dp, nranks):
    """Every rank's ShardInfo, or None when the split is refused."""
    out = []
    for r in range(nranks):
        rc, si = shard_query_desc(dp, r, nranks)
        if rc != 0:
            assert rc == ERR_UNSUPPORTED, (r, nranks, rc)
            return None
        out.append(si)
    return out


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_partition_is_consistent(c):
    sw, sh, nw, nh, ch, ti, to, kw = c
    ran = 0
    with Descriptor(c) as dd:
        for n in RANKS:
            bs = bands(dd.ptr, n)
            if bs is None:
                continue
            ran += 1
            assert bs[0].src_row0 == 0 and bs[0].dst_row0 == 0
            assert bs[-1].src_row0 + bs[-1].src_rows == sh and bs[-1].dst_row0 + bs[-1].dst_rows == nh
            assert bs[0].halo_up == 0 and bs[-1].halo_down == 0
            for r, b in enumerate(bs):
                assert b.src_rows > 0 and b.dst_rows > 0
                assert (b.src_row0, b.dst_row0) == (sh * r // n, nh * r // n)
                if r + 1 < n:
                    assert bs[r + 1].src_row0 == b.src_row0 + b.src_rows
                    assert bs[r + 1].dst_row0 == b.dst_row0 + b.dst_rows
                assert b.need_row0 == b.src_row0 - b.halo_up
                assert b.need_rows == b.halo_up + b.src_rows + b.halo_down
                assert 0 <= b.need_row0 and b.need_row0 + b.need_rows <= sh
                assert b.halo_up >= 0 and b.halo_down >= 0
                if r > 0:
                    assert b.halo_up <= bs[r - 1].src_rows
                if r + 1 < n:
                    assert b.halo_down <= bs[r + 1].src_rows
                # `need` is the footprint joined with the own band
                lo, hi = brute_span(dd.desc.v, b.dst_row0, b.dst_rows)
                assert b.need_row0 == min(lo, b.src_row0)
                assert b.need_row0 + b.need_rows - 1 == max(hi, b.src_row0 + b.src_rows - 1)
    assert ran >= 1


def test_too_many_ranks_are_refused_without_a_device():
    """48 x 27 -> 8 bands of 3 rows with a 12-tap kernel: the halos reach past the neighbours' bands."""
    c = (96, 54, 48, 27, 4, np.uint8, np.uint8, {})
    with Descriptor(c) as dd:
        assert bands(dd.ptr, 2) is not None
        for n in (18, 27, 54, 55, 1000):
            assert bands(dd.ptr, n) is None, n


def test_need_is_the_span_of_the_clamped_taps_at_full_size():
    """8K -> 4K RGBA: a band of 540 rows (8 ranks) reads its 1080 own rows plus 5 rows beyond each side."""
    c = (7680, 4320, 3840, 2160, 4, np.uint8, np.uint8, {})
    with Descriptor(c) as dd:
        bs = bands(dd.ptr, 8)
        for r, b in enumerate(bs):
            assert (b.src_rows, b.dst_rows) == (540, 270)
            assert (b.halo_up, b.halo_down) == (0 if r == 0 else 5, 0 if r == 7 else 5)


@pytest.mark.parametrize("c", CASES, ids=case_id)
def test_need_holds_every_source_row_the_band_reads(c):
    sw, sh, nw, nh, ch, ti, to, kw = c
    src = o.lcg_image(sh, sw, ch, ti, seed=23)
    with Descriptor(c) as dd:
        full = port_resize(dd.ptr, src, nw, nh, to)
        for n in RANKS:
            bs = bands(dd.ptr, n)
            if bs is None:
                continue
            for b in bs:
                rows = slice(b.need_row0, b.need_row0 + b.need_rows)
                for poison in _poisons(src.dtype):
                    bad = np.full_like(src, poison)
                    bad[rows] = src[rows]
                    got = port_resize(dd.ptr, bad, nw, nh, to)
                    d = slice(b.dst_row0, b.dst_row0 + b.dst_rows)
                    assert np.array_equal(full[d].view(np.uint8), got[d].view(np.uint8)), (n, b.dst_row0, poison)


def test_tall_plan_bands():
    """A plan of 70001 destination rows: one band is too tall for the kernels' grid, two are not."""
    c = (6, 35000, 4, 70001, 1, np.uint8, np.uint8, {})
    with Descriptor(c) as dd:
        rc, _ = shard_query_desc(dd.ptr, 0, 1)
        assert rc == ERR_UNSUPPORTED
        bs = bands(dd.ptr, 2)
        assert bs is not None and [b.dst_rows for b in bs] == [35000, 35001]
        bs = bands(dd.ptr, 3)
        assert bs is not None


def test_refusals_without_a_device():
    L = ab.lib()
    vp, i, sz = C.c_void_p, C.c_int, C.c_size_t
    L.lancirb200_shard_query.argtypes = [vp, i, i, vp]
    L.lancirb200_shard_query_desc.argtypes = [vp, i, i, vp]
    L.lancirb200_shard_workspace_bytes.argtypes = [vp, i, i, vp]
    L.lancirb200_resize_sharded.argtypes = [vp, vp, i, i, vp, sz, vp, sz, vp, vp]
    L.lancirb200_resize_sharded_host.argtypes = [vp, vp, i, i, vp, sz, vp, sz]
    L.lancirb200_resize_sharded_local.argtypes = [vp, i, vp, sz, vp, sz, vp, vp]
    L.lancirb200_plan_set_option.argtypes = [vp, i, i]
    si, n = ShardInfo(), C.c_size_t()
    buf = np.zeros(64, np.uint8)
    p = buf.ctypes.data
    assert L.lancirb200_shard_query_desc(None, 0, 2, C.byref(si)) == ERR_BAD_ARG
    assert L.lancirb200_shard_query(None, 0, 2, C.byref(si)) == ERR_BAD_ARG
    assert L.lancirb200_shard_workspace_bytes(None, 0, 2, C.byref(n)) == ERR_BAD_ARG
    assert L.lancirb200_resize_sharded(None, p, 0, 2, p, 4, p, 4, p, None) == ERR_BAD_ARG
    assert L.lancirb200_resize_sharded_host(None, p, 0, 2, p, 4, p, 4) == ERR_BAD_ARG
    assert L.lancirb200_resize_sharded_local(None, 2, p, 4, p, 4, p, None) == ERR_BAD_ARG
    assert L.lancirb200_plan_set_option(None, ab.api.OPT_OVERLAP_HALO, 0) == ERR_BAD_ARG
    with Descriptor((96, 54, 48, 27, 4, np.uint8, np.uint8, {})) as dd:
        assert L.lancirb200_shard_query_desc(dd.ptr, 0, 2, None) == ERR_BAD_ARG
        for rank, nranks in ((-1, 2), (2, 2), (0, 0), (0, -3), (5, 4)):
            assert shard_query_desc(dd.ptr, rank, nranks)[0] == ERR_BAD_ARG, (rank, nranks)
        assert shard_query_desc(dd.ptr, 0, 28)[0] == ERR_UNSUPPORTED      # a rank without destination rows
        assert shard_query_desc(dd.ptr, 1, 1)[0] == ERR_BAD_ARG
        assert shard_query_desc(dd.ptr, 0, 1)[0] == 0


def test_multi_gpu_worker_cases_split_at_every_rank_count():
    """tests/lancir_sharded_worker.py's host-side setup without GPUs: every case's descriptor builds with the
    worker's own type codes and splits at 2, 4 and 8 ranks; the list holds pairs whose rows travel both ways
    (the mailboxes, both slots) and pairs whose rows travel one way only (NCCL) at every rank count."""
    import lancir_sharded_worker as w
    for n in (2, 4, 8):
        both = one_way = 0
        for case in w.CASES:
            h, dp = w.descriptor(case)
            try:
                bs = bands(dp, n)
                assert bs is not None, (case[:5], n)
                for a, b in zip(bs, bs[1:]):
                    both += a.halo_down > 0 and b.halo_up > 0
                    one_way += (a.halo_down > 0) != (b.halo_up > 0)
            finally:
                ab.host_lib().lancirb200_host_desc_free(h)
        assert both and one_way, (n, both, one_way)
