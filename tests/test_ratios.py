"""Large downscale ratios, tiny destinations and extreme upscales without a GPU: the planner against
upstream's recorded plans, the C port (the GPU tests' fallback reference) against upstream on the strip
cases, and the generic kernel's shared-memory layout (avir_b200/csrc/pass_config.h, the engine's own
code) through tests/emul/config_emul.cpp.  The GPU side is tests/test_gpu_ratios.py."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import cases as cs
import oracle_ref as o
import plan_util as pu
from test_gpu_parity import MEDIUM
from test_gpu_ratios import LADDER, REFUSED, SURFACE, THUMBS, TINY, UPSCALES, strip

u8, u16, f32 = np.uint8, np.uint16, np.float32
needs_ref = pytest.mark.skipif(not o.have_ref(), reason="oracle/_ref not built")

H100_SMEM_OPTIN = 232448  # cudaDevAttrMaxSharedMemoryPerBlockOptin of an H100: 227 KiB
PREFERRED = 100 * 1024    # pass_config.h, kGenericSmemPreferred
CAND = [1024, 768, 512, 384, 256, 192, 128, 96, 64, 48, 32, 24, 16, 12, 8, 4, 2, 1]

# full-size BASELINE.json chains (configs[1..4])
BASELINE = [
    (0, 1920, 1080, 3840, 2160, 4, u8, u8, 8, {}),
    (2, 7680, 4320, 3840, 2160, 4, f32, f32, 16, {}),
    (1, 7680, 4320, 3840, 2160, 4, f32, f32, 16, {}),
    (1, 16384, 16384, 4096, 4096, 4, u16, u16, 16, {}),
    (2, 7680, 4320, 1920, 1080, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),
]
REFUSED_CASES = [c[:10] for c in REFUSED]


def _geometry(cases):
    """One case per distinct plan geometry (the channel count does not change a plan)."""
    seen, out = set(), []
    for c in cases:
        fp, sw, sh, nw, nh, ch, ti, to, rb, kw = c
        key = (fp % 3, sw, sh, nw, nh, np.dtype(ti).name, np.dtype(to).name, rb, json.dumps(kw, sort_keys=True))
        if key not in seen:
            seen.add(key)
            out.append(c)
    return out


PLANNED = _geometry(LADDER + THUMBS + TINY + SURFACE + UPSCALES + REFUSED_CASES)


@needs_ref
@pytest.mark.parametrize("case", PLANNED, ids=cs.case_id)
def test_planner_matches_upstream_at_extreme_ratios(case):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rk = cs.ref_kwargs(kw)
    rp, _ = o.ref_plan(np.zeros((sh, sw, ch), ti), nw, nh, to, fpclass=fp % 3, resbits=rb, **rk)
    mp = pu.host_plan(fp % 3, sw, sh, nw, nh, ch, ti, to, k=rk["k"], resbits=rb, ox=rk["ox"], oy=rk["oy"],
                      gamma=rk["gamma"], buildmode=rk["buildmode"], params=rk["params"])
    assert pu.compare_axis(mp["H"], rp["H"]) == []
    assert pu.compare_axis(mp["V"], rp["V"]) == []


STRIPS = [c for c in LADDER if c[5] in (1, 4)] + SURFACE


@needs_ref
@pytest.mark.parametrize("case", STRIPS, ids=cs.case_id)
def test_port_matches_upstream_on_strips(case):
    src = cs.make_input(case)
    assert cs.value_mismatch(cs.ref_output(case, src), cs.port_output(case, src)[0]) == 0


# ---- the generic kernel's layout (pass_config.h) ------------------------------------------------------

@pytest.fixture(scope="module")
def cfg():
    from avir_b200 import build as b
    lib = C.CDLL(b.build_config_emul())
    lib.config_emul_generic.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong,
                                        C.POINTER(C.c_longlong)]
    lib.config_emul_generic.restype = None
    lib.config_emul_max_span.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    lib.config_emul_max_span.restype = C.c_int
    return lib


def configs(lib, case, channels=None, max_smem=H100_SMEM_OPTIN):
    """{"row": (lines, tile, span_a, span_b, pitch, smem), "col": ...} of the case's whole-image passes."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, kw.get("k", 0.0), v)
    try:
        out = {}
        for axis, name, n in ((0, "row", nw), (1, "col", nh)):
            r = (C.c_longlong * 6)()
            lib.config_emul_generic(dp, axis, channels or ch, 0, n, max_smem, r)
            out[name] = tuple(r)
            out[name + "_old"] = _old_rule(lib, dp, axis, channels or ch, n)
        return out
    finally:
        rs.free_descriptor(h)


def _old_rule(lib, dp, axis, ch, n):
    """(lines, tile, smem) of the rule that sized both buffers by the larger span and stopped at one
    output per tile, whether or not it fit."""
    lines = max(1, 64 // ch)
    pitch = (lines * ch) | 1
    for t in CAND:
        smem = 2 * lib.config_emul_max_span(dp, axis, t, 0, n) * pitch * 4
        if smem <= PREFERRED or t == 1:
            return lines, t, smem


FITTING = [c for c in LADDER + THUMBS + TINY + SURFACE + UPSCALES]


@pytest.mark.parametrize("case", FITTING, ids=cs.case_id)
def test_every_large_ratio_case_fits_the_generic_kernel(cfg, case):
    c = configs(cfg, case)
    for p in ("row", "col"):
        lines, t, sa, sb, pitch, smem = c[p]
        assert smem <= H100_SMEM_OPTIN, (p, c[p])
        assert pitch == (lines * case[5]) | 1 and smem == (sa + sb) * pitch * 4
        if c[p + "_old"][2] <= H100_SMEM_OPTIN:   # what fit before keeps its layout
            assert (lines, t) == c[p + "_old"][:2] and smem <= c[p + "_old"][2]


@pytest.mark.parametrize("case", REFUSED_CASES, ids=cs.case_id)
def test_only_long_four_channel_lines_to_very_few_pixels_are_refused(cfg, case):
    """The documented bound: a 4-channel line of 16384 px to one pixel does not fit one output of one
    line (5 floats per source position); the same line with 1..3 channels does, and so does a
    4-channel line of 11264 px."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    c = configs(cfg, case)
    p = "row" if sw > nw else "col"
    assert c[p][0] == 1 and c[p][1] == 1 and c[p][5] > H100_SMEM_OPTIN, c[p]
    for ch2 in (1, 2, 3):
        assert configs(cfg, case, channels=ch2)[p][5] <= H100_SMEM_OPTIN
    ok = (fp, 11264, 4, 1, 4, 4, ti, to, rb, kw) if p == "row" else (fp, 4, 11264, 4, 1, 4, ti, to, rb, kw)
    assert configs(cfg, ok)[p][5] <= H100_SMEM_OPTIN


def test_the_bound_of_a_four_channel_line(cfg):
    """The 4-channel line length past which one output to one pixel no longer fits, on an H100: between
    11 264 and 11 776 source pixels (include/avirb200.h, avirb200_plan_create: about 11 600)."""
    fits = {n: configs(cfg, (1, n, 4, 1, 4, 4, u8, u8, 8, {}))["row"][5] <= H100_SMEM_OPTIN for n in (11264, 11776)}
    assert fits == {11264: True, 11776: False}


@pytest.mark.parametrize("case", cs.SMALL_CASES + MEDIUM + BASELINE, ids=cs.case_id)
def test_existing_layouts_are_unchanged(cfg, case):
    """Every case that fit before keeps its lines per block and tile length; only the buffers shrink to
    their own spans."""
    c = configs(cfg, case)
    for p in ("row", "col"):
        lines, t, sa, sb, pitch, smem = c[p]
        ol, ot, osm = c[p + "_old"]
        assert osm <= H100_SMEM_OPTIN, (p, c)
        assert (lines, t) == (ol, ot) and smem <= osm, (p, c)
