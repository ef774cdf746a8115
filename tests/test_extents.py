"""Images past 16- and 32-bit extents without a GPU: the premises of tests/test_gpu_extents.py and the host
arithmetic at those sizes.

* The generic kernel's layout (pass_config.h through tests/emul/config_emul.cpp): the tall cases really get
  one line per block, or 16 lines per block with more than 65535 blocks.  If the layout rule changes, this
  fails before the GPU test quietly stops crossing the grid limit.
* The C port (the GPU tests' fallback reference) against upstream on the tall and wide cases.
* avirb200_window_query_desc / lancirb200_window_query_desc on the huge shapes: the tiling the GPU test
  uses covers the destination, every footprint holds its tile's own source span and every buffer of a
  tile's window call stays far below 2^31 bytes.
* avirb200_shard_layout_desc for plans whose workspace passes 4 GiB, against ws_layout's arithmetic
  restated in Python integers: no size is cut to 32 bits."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import oracle_ref as o
import plan_util as pu
from test_gpu_extents import (BIG, ERRD_BIG, LANCIR_BIG, LPB1_COL, LPB1_ROW, STRIP, TALL, WINDOW_LIMIT, tile_buffers,
                              tiles)
from test_lancir_window import Descriptor
from test_lancir_window import query_desc as lancir_query_desc
from test_ratios import configs
from test_ratios import cfg  # noqa: F401  (the config_emul fixture)
from test_sharded_errd import mailbox_bytes, shard_layout, shard_workspace_bytes
from test_window import window_query_desc

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
needs_ref = pytest.mark.skipif(not o.have_ref(), reason="oracle/_ref not built")
GRID_Y = 65535  # blocks a launch may have along y


def line_blocks(case, c, p):
    """Blocks of lines the generic kernel needs for pass p ("row": the source rows, "col": the destination
    columns) at layout c."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    lines = sh if p == "row" else nw
    return -(-lines // c[p][0])


@pytest.mark.parametrize("case,p", [(LPB1_COL, "col"), (LPB1_ROW, "row")], ids=["column-pass", "row-pass"])
def test_long_lines_to_few_pixels_get_one_line_per_block(cfg, case, p):
    c = configs(cfg, case)
    assert c[p][0] == 1 and c[p][1] == 1, c[p]
    assert line_blocks(case, c, p) == 66000 > GRID_Y


def test_the_tall_strip_needs_more_than_65535_blocks_of_16_lines(cfg):
    c = configs(cfg, STRIP)
    assert c["row"][0] == 16, c["row"]
    assert line_blocks(STRIP, c, "row") == 68750 > GRID_Y
    # the vertical chain holds a filtered 2X upsample (step kind 1), which no streaming or tile chain serves
    # (tests/test_gpu_extents.py checks that the plan's passes qualify for neither)
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = STRIP
    plan = pu.host_plan(fp, sw, sh, nw, nh, ch, ti, to, resbits=rb, buildmode=0)
    assert any(s["kind"] == 1 for s in plan["V"]["steps"]), [s["kind"] for s in plan["V"]["steps"]]


@needs_ref
@pytest.mark.parametrize("name", ["strip-1.1M", "stream-tall", "tile-wide", "rgb-wide", "gray-tall"])
def test_port_matches_upstream_on_tall_and_wide_images(name):
    case = TALL[name]
    src = cs.make_input(case, seed=17)
    want = o.ref_resize(src, *case[3:5], case[7], fpclass=case[0], resbits=case[8], nthreads=8,
                        **cs.ref_kwargs(case[9]))
    assert cs.count_mismatch(want, cs.port_output(case, src)[0]) == 0


def check_tiling(nw, nh, sw, sh, ch, ti, to, query):
    covered = np.zeros((nh, nw), np.int8)
    for win in tiles(nw, nh):
        x0, y0, w, h = win
        rc, fi = query(win)
        assert rc == 0, win
        assert 0 <= fi.src_x0 and fi.src_x0 + fi.src_w <= sw and 0 <= fi.src_y0 and fi.src_y0 + fi.src_h <= sh, win
        # the tile's own source span: the source pixels its destination pixels cover
        own_x = (x0 * sw // nw, min(sw, -(-(x0 + w) * sw // nw)))
        own_y = (y0 * sh // nh, min(sh, -(-(y0 + h) * sh // nh)))
        assert fi.src_x0 <= own_x[0] and fi.src_x0 + fi.src_w >= own_x[1], (win, own_x)
        assert fi.src_y0 <= own_y[0] and fi.src_y0 + fi.src_h >= own_y[1], (win, own_y)
        assert max(tile_buffers(fi, win, ch, ti, to)) < WINDOW_LIMIT // 2, win
        covered[y0:y0 + h, x0:x0 + w] += 1
    assert (covered == 1).all()


@pytest.mark.parametrize("name", list(BIG))
def test_window_tiling_of_the_big_cases(name):
    case = BIG[name]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, v)
    try:
        check_tiling(nw, nh, sw, sh, ch, ti, to, lambda win: window_query_desc(dp, win))
    finally:
        rs.free_descriptor(h)


def test_window_tiling_of_the_big_lancir_case():
    sw, sh, nw, nh, ch, ti = LANCIR_BIG
    with Descriptor((sw, sh, nw, nh, ch, ti, ti, {})) as d:
        check_tiling(nw, nh, sw, sh, ch, ti, ti, lambda win: lancir_query_desc(d.ptr, win))


# plans whose one-rank workspace passes 4 GiB: double source and destination, error diffusion
SHARD_BIG = [
    (1, 23200, 23200, 11600, 11600, 4, f64, f64, 16, {}),
    (4, 33000, 33000, 16500, 16500, 4, u8, u8, 8, {}),
    ERRD_BIG,
]


@pytest.mark.parametrize("nranks", [1, 2, 3])
@pytest.mark.parametrize("case", SHARD_BIG, ids=cs.case_id)
def test_shard_layout_past_4_gib(case, nranks):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    errd = fp >= 3 and np.dtype(to).kind != "f"
    sizes = []
    for rank in range(nranks):
        r, ws, box, si = shard_layout(case, rank, nranks)
        assert r == 0, (rank, ab.lib().avirb200_last_error())
        assert ws == shard_workspace_bytes(si, sw, nw, ch, np.dtype(ti) == f64, np.dtype(to) == f64, errd), rank
        assert box == mailbox_bytes(si, nw, ch, errd, 2), rank
        sizes.append(ws)
    if nranks == 1:
        assert sizes[0] > 1 << 32, sizes
