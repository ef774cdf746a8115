"""The C-ABI library loads on a CPU-only box, exports every symbol include/avirb200.h
declares, and refuses to compute without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    txt = open(os.path.join(ROOT, "include", "avirb200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    names = re.findall(r"\b((?:avirb200|lancirb200)_[a-z0-9_]+)\s*\(", txt)
    return sorted(set(names))


def test_every_declared_symbol_is_exported():
    lib = ab.lib()
    names = declared_functions()
    assert len(names) >= 23
    for n in names:
        assert hasattr(lib, n), "libavirb200.so does not export " + n


def test_status_strings():
    lib = ab.lib()
    assert lib.avirb200_status_string(0) == b"ok"
    for code in range(-6, 0):
        assert lib.avirb200_status_string(code) not in (b"ok", b"unknown status")


def test_bad_arguments_are_rejected_before_touching_cuda():
    lib = ab.lib()
    out = C.c_void_p()
    assert lib.avirb200_plan_create(None, C.byref(out)) == -1
    assert lib.lancirb200_plan_create(None, C.byref(out)) == -1
    info = (C.c_int * 8)()
    assert lib.avirb200_shard_query_desc(None, 0, 1, info) == -1


class _LancirAxis(C.Structure):
    _fields_ = [("src_len", C.c_int32), ("dst_len", C.c_int32), ("kernel_len", C.c_int32), ("nphases", C.c_int32),
                ("taps", C.c_void_p), ("src_pos", C.c_void_p), ("phase", C.c_void_p)]


class _LancirDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("src_w", "src_h", "dst_w", "dst_h", "channels", "in_type", "out_type")] + [
        ("out_mul", C.c_float), ("is_unity_mul", C.c_int32), ("clamp_max", C.c_float),
        ("v", _LancirAxis), ("h", _LancirAxis)]


def test_lancir_failures_are_reported_by_last_error():
    """avirb200_last_error() reports a LANCIR failure with LANCIR's own message, not an older one."""
    lib = ab.lib()
    out = C.c_void_p()
    assert lib.avirb200_plan_create(None, C.byref(out)) == -1
    assert lib.avirb200_last_error() == b"null argument"
    desc = _LancirDesc(src_w=8, src_h=8, dst_w=4, dst_h=4, channels=5)
    assert lib.lancirb200_plan_create(C.byref(desc), C.byref(out)) == -1
    assert lib.avirb200_last_error() == b"channels must be 1..4"


@pytest.mark.skipif(ab.device_count() > 0, reason="checks the no-GPU behaviour")
def test_no_cpu_fallback_without_gpu():
    """Without a device the product must fail loudly, never compute on the host."""
    case = cs.SMALL_CASES[0]
    src = cs.make_input(case)
    with pytest.raises(ab.AvirB200Error) as e:
        cs.gpu_output(case, src)
    assert "no usable CUDA device" in str(e.value) or "CUDA" in str(e.value)
    r, _ = ab.CLancIR().resizeImage(np.zeros((8, 8, 4), np.uint8), 4, 4)
    assert r == 0  # upstream's error convention (lancir.h:382-383)


def test_descriptor_is_built_without_gpu():
    case = cs.SMALL_CASES[2]
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = cs.resizer_and_vars(case)
    h, dp, modes = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, v)
    assert dp and modes[0] in (0, 1) and modes[1] in (0, 1)
    rs.free_descriptor(h)


def test_lancir_argument_errors_follow_upstream():
    # lancir.h:392-408: bad sizes / la < 2 -> 0
    r, _ = ab.CLancIR().resizeImage(np.zeros((8, 8, 4), np.uint8), 4, 4, ab.CLancIRParams(la=1.5))
    assert r == 0


def test_plan_options_reject_bad_arguments():
    lib = ab.lib()
    lib.avirb200_plan_set_option.argtypes = [C.c_void_p, C.c_int, C.c_int]
    assert lib.avirb200_plan_set_option(None, 0, 0) == -1
    assert lib.avirb200_resize_device_batch(None, 0, None, 0, None, 0, None, None) == -1
    assert lib.avirb200_resize_sharded_host(None, None, 0, 1, None, 0, None, 0) == -1


def test_host_generator_is_the_survey_generator():
    """bench.py's synthetic input (C loop in the host driver library) == the SURVEY 8(d) xorshift32
    generator as the tests spell it in Python."""
    import oracle_ref as o
    hl = ab.host_lib()
    hl.avirb200_host_fill_xorshift32.argtypes = [C.c_void_p, C.c_size_t, C.c_uint32, C.c_int]
    hl.avirb200_host_fill_xorshift32.restype = C.c_uint32
    for dt, code in ((np.uint8, 0), (np.uint16, 1), (np.float32, 2)):
        want = o.xorshift32_image(7, 11, 3, dt, seed=12345)
        got = np.empty((7, 11, 3), dt)
        hl.avirb200_host_fill_xorshift32(got.ctypes.data, got.size, 12345, code)
        assert np.array_equal(want.view(np.uint8), got.view(np.uint8)), dt


def test_lancir_rejects_double_buffers():
    with pytest.raises(ab.AvirB200Error):
        ab.CLancIR().resizeImage(np.zeros((8, 8, 4), np.float64), 4, 4)
    with pytest.raises(ab.AvirB200Error):
        ab.CLancIR().resizeImage(np.zeros((8, 8, 4), np.uint8), 4, 4, out_dtype=np.float64)


def test_vars_outputs_are_filled_on_plan_cache_hits():
    """A second identical call (served from the front-end's plan cache) reports the same
    informational Vars outputs as the first."""
    hl = ab.host_lib()
    hl.avirb200_host_vars_probe.argtypes = [C.c_int] * 4 + [C.c_void_p]
    out = (C.c_double * 8)()
    assert hl.avirb200_host_vars_probe(64, 48, 100, 75, out) == 0
    first, second = list(out)[:4], list(out)[4:]
    assert first == second and first[0] == 4 and first[2] > 0.0 and first[3] >= 0
