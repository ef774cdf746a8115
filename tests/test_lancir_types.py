"""CLancIR with double and uint32_t buffers, without a GPU (upstream lancir.h:373-381 takes uint8_t, uint16_t,
float, double and uint32_t, the last treated as uint16_t).

* The oracle's C port (lancir_types_port_resize over avir_port.c's passes), run on the descriptor the front-end builds, equals upstream
  compiled in-tree on every type pair involving double or uint32_t, on random and value-domain sources
  (NaN positions must match, payloads need not: cases.value_mismatch).
* The committed types_*.npz fixtures (upstream's output) equal the port where oracle/_ref is absent.
* The descriptor's out_mul / is_unity_mul / clamp_max are upstream's formulas (lancir.h:526-533).
* A NaN in the (NewWidth * C) & 3 half-up tail stores x86's (int)NaN: 2147483648 as uint32_t, 0 as u8 / u16.
* The C++ front-end compiles with double and uint32_t and refuses other types at compile time; the C ABI
  and the host entry points refuse type codes they do not take.
"""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs
import lancir_types_oracle as lo
import oracle_ref as o

u8, u16, f32, f64, u32 = np.uint8, np.uint16, np.float32, np.float64, np.uint32
TYPES = (u8, u16, f32, f64, u32)
NEW = (f64, u32)
NEW_PAIRS = [(ti, to) for ti in TYPES for to in TYPES if ti in NEW or to in NEW]
ERR_BAD_ARG = -1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not lo.have_ref(), reason="needs oracle/_ref (upstream CLancIR)")

# double sources: beyond float's range (+-Inf once narrowed), non-finite, inside float's subnormal range,
# below it (+-0 once narrowed), -0.0, above 1
F64_VALUES = [1e39, -1e39, np.inf, -np.inf, np.nan, 1e-40, -3e-42, 2.0 ** -149, 1e-46, -1e-50, 5e-324, -0.0,
              1.5, 3.0, 70000.0]
F64_TINY = [1e-40, -3e-42, 2.0 ** -149, 2.0 ** -130, 1e-46, -1e-50, 5e-324, -0.0, 0.0]
# uint32_t sources: the u16 maximum, just past it, past float's exact integers, the type's maximum
U32_VALUES = [65535, 65536, 2 ** 24 + 1, 0xFFFFFFFF, 2 ** 24, 0, 1000000]

# (sw, sh, nw, nh, channels, CLancIRParams fields): 1-4 channels, la 2 / 3 / 5, k = 2 / 3, upsizing,
# explicit and negative k, offsets
GEOMS = [
    (96, 54, 48, 27, 4, {}),
    (64, 48, 103, 77, 3, {}),
    (77, 51, 47, 29, 2, {"la": 2.0}),
    (60, 45, 20, 15, 1, {"la": 5.0}),
    (50, 30, 70, 45, 4, {"kx": 0.7, "ky": -0.66, "ox": 0.25, "oy": 0.1}),
    (77, 51, 47, 29, 3, {"kx": -1.3, "ky": 2.2, "ox": -0.4}),
]

# (sw, sh, nw, nh, channels, Tin, Tout, source kind): every new type as the source and as the destination,
# 1-4 channels, random and value-domain sources, and one NaN in a uint32_t row tail
TYPE_FIXTURES = [
    (96, 54, 48, 27, 4, f64, f64, "random"),
    (64, 48, 103, 77, 3, u32, u32, "random"),
    (77, 51, 47, 29, 2, u8, f64, "random"),
    (60, 40, 40, 27, 1, f64, u8, "random"),
    (50, 30, 33, 17, 4, u16, u32, "random"),
    (77, 51, 47, 29, 3, u32, f32, "random"),
    (64, 48, 32, 24, 4, f64, u32, "values"),
    (64, 48, 33, 23, 1, u32, f64, "values"),
    (64, 48, 35, 23, 3, f64, f32, "values"),
    (8, 2, 3, 2, 1, f64, u32, "nan_tail"),
]


def pid(t):
    return np.dtype(t).name


def type_image(h, w, c, dtype, seed):
    """A seeded random image: the oracle's generator for u8 / u16 / float / double (double values are not
    representable in float: the (float) cast rounds), uint32_t drawn as u16 codes (upstream's range)."""
    if np.dtype(dtype) == np.uint32:
        return o.lcg_image(h, w, c, np.uint16, seed=seed).astype(np.uint32)
    return o.lcg_image(h, w, c, dtype, seed=seed)


def value_source(h, w, c, dtype, seed):
    """A value-domain source of a new type.  double: sparse F64_VALUES on a [0, 1) background in the top
    half, a band of F64_TINY values (outputs in float's subnormal range) below.  uint32_t: blocks of
    U32_VALUES on a u16 background."""
    rng = np.random.default_rng(seed)
    if np.dtype(dtype) == np.float64:
        img = rng.random((h, w, c))
        n = max(8, h * w * c // 40)
        img[:h // 2].reshape(-1)[rng.integers(0, (h // 2) * w * c, n)] = [F64_VALUES[i % len(F64_VALUES)]
                                                                         for i in range(n)]
        img[h // 2:] = rng.choice(F64_TINY, (h - h // 2, w, c))
        return img
    img = type_image(h, w, c, u32, seed)
    for i in range(max(4, h * w // 60)):
        y, x = int(rng.integers(0, h)), int(rng.integers(0, w))
        img[y:y + 3, x:x + 3, int(rng.integers(0, c))] = U32_VALUES[i % len(U32_VALUES)]
    return img


def fixture_source(c, seed):
    sw, sh, nw, nh, ch, ti, to, kind = c
    if kind == "random":
        return type_image(sh, sw, ch, ti, seed)
    if kind == "values":
        return value_source(sh, sw, ch, ti, seed)
    assert kind == "nan_tail"
    src = type_image(sh, sw, ch, ti, seed)
    src[0, 3, 0] = np.nan
    return src


port_resize = lo.port_resize


# ---- the port against upstream -----------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("g", GEOMS, ids=lambda g: "%dx%d-%dx%d-c%d" % g[:5] + "".join(
    "-%s%s" % kv for kv in sorted(g[5].items())))
@pytest.mark.parametrize("ti,to", NEW_PAIRS, ids=lambda t: pid(t))
def test_port_matches_upstream(ti, to, g):
    sw, sh, nw, nh, ch, kw = g
    src = type_image(sh, sw, ch, ti, seed=sw + ch)
    r, want = lo.lancir_ref(src, nw, nh, to, kw)
    assert r == nh
    assert cs.value_mismatch(want, port_resize(src, nw, nh, to, kw)) == 0


@needs_ref
@pytest.mark.parametrize("ch", [1, 2, 3, 4])
@pytest.mark.parametrize("to", TYPES, ids=pid)
@pytest.mark.parametrize("ti", NEW, ids=pid)
def test_port_value_domain_matches_upstream(ti, to, ch):
    for sw, sh, nw, nh, kw in [(70, 50, 33, 23, {}), (40, 30, 61, 47, {"la": 2.0}),
                               (70, 50, 29, 19, {"kx": -2.1, "ky": 2.6, "ox": 0.3})]:
        src = value_source(sh, sw, ch, ti, seed=ch + sw)
        r, want = lo.lancir_ref(src, nw, nh, to, kw)
        assert r == nh
        got = port_resize(src, nw, nh, to, kw)
        assert cs.value_mismatch(want, got) == 0, (sw, sh, nw, nh, kw)
    if ti == f64 and to in (f32, f64):   # the tiny band's outputs stay subnormal
        tiny = np.abs(got[-nh // 3:].astype(np.float64))
        assert ((tiny > 0) & (tiny < 2.0 ** -126)).any()


# ---- fixtures ---------------------------------------------------------------------------------------------

def fixture_files():
    return sorted(f for f in os.listdir(cs.GOLDEN) if f.startswith("types_") and f.endswith(".npz"))


def test_fixtures_cover_the_new_types():
    zs = [np.load(os.path.join(cs.GOLDEN, f)) for f in fixture_files()]
    assert len(zs) == len(TYPE_FIXTURES)
    for t in NEW:
        assert any(z["src"].dtype == t for z in zs) and any(z["out"].dtype == t for z in zs), pid(t)
    assert {z["src"].shape[2] for z in zs} == {1, 2, 3, 4}
    assert any(str(z["kind"]) == "nan_tail" for z in zs)


@pytest.mark.parametrize("f", fixture_files())
def test_port_matches_fixture(f):
    z = np.load(os.path.join(cs.GOLDEN, f))
    sw, sh, nw, nh = [int(v) for v in z["geom"]]
    got = port_resize(z["src"], nw, nh, z["out"].dtype)
    assert cs.value_mismatch(z["out"], got) == 0


# ---- the descriptor's output constants --------------------------------------------------------------------

def upstream_constants(ti, to):
    """lancir.h:526-533 in float arithmetic: (OutMul, IsUnityMul, Clamp)."""
    in_f, out_f = np.dtype(ti).kind == "f", np.dtype(to).kind == "f"
    si, so = np.dtype(ti).itemsize, np.dtype(to).itemsize
    clamp = np.float32(255.0 if so == 1 else 65535.0)
    mul = (np.float32(1.0) if out_f else clamp) / np.float32(1.0 if in_f else (255.0 if si == 1 else 65535.0))
    return np.float32(mul), int((in_f and out_f) or (in_f == out_f and si == so)), clamp


@pytest.mark.parametrize("to", TYPES, ids=pid)
@pytest.mark.parametrize("ti", TYPES, ids=pid)
def test_descriptor_constants(ti, to):
    with lo.Descriptor(40, 30, 20, 15, 4, ti, to) as d:
        mul, unity, clamp = upstream_constants(ti, to)
        assert (d.desc.in_type, d.desc.out_type) == (lo.code(ti), lo.code(to))
        assert np.float32(d.desc.out_mul) == mul
        assert d.desc.is_unity_mul == unity
        assert np.float32(d.desc.clamp_max) == clamp


def test_descriptor_constants_of_the_new_pairs():
    """The consequences upstream's formulas have for uint32_t and double, spelled out."""
    want = {(u32, u32): (1.0, 1), (f64, f64): (1.0, 1), (f64, f32): (1.0, 1), (f32, f64): (1.0, 1),
            (u16, u32): (1.0, 0), (u32, u16): (1.0, 0), (u8, u32): (257.0, 0), (f64, u32): (65535.0, 0),
            (u32, f64): (np.float32(1.0) / np.float32(65535.0), 0), (u32, u8): (np.float32(255.0) / np.float32(65535.0), 0)}
    for (ti, to), (mul, unity) in want.items():
        with lo.Descriptor(40, 30, 20, 15, 4, ti, to) as d:
            assert (np.float32(d.desc.out_mul), d.desc.is_unity_mul) == (np.float32(mul), unity), (pid(ti), pid(to))
            assert d.desc.clamp_max == (255.0 if to == u8 else 65535.0)


# ---- a NaN in the half-up tail ------------------------------------------------------------------------------

NAN_TAIL = TYPE_FIXTURES[-1]


@pytest.mark.parametrize("to,want", [(u32, 2147483648), (u16, 0), (u8, 0)], ids=["uint32", "uint16", "uint8"])
def test_nan_in_the_tail(to, want):
    sw, sh, nw, nh, ch, ti, _, kind = NAN_TAIL
    assert kind == "nan_tail" and (nw * ch) & 3 == nw * ch   # every element is in the tail
    src = fixture_source(NAN_TAIL, seed=400 + len(TYPE_FIXTURES) - 1)
    got = port_resize(src, nw, nh, to)
    assert (got == want).all(), got
    if lo.have_ref():
        r, ref = lo.lancir_ref(src, nw, nh, to)
        assert r == nh and (ref == want).all(), ref
    if to == u32:
        z = np.load(os.path.join(cs.GOLDEN, "types_%02d.npz" % (len(TYPE_FIXTURES) - 1)))
        assert np.array_equal(z["src"], src, equal_nan=True) and (z["out"] == want).all()


# ---- refusals ----------------------------------------------------------------------------------------------

def test_lancir_plan_create_refuses_other_type_codes():
    L = ab.lib()
    for field in ("in_type", "out_type"):
        for code in (5, -1, 1 << 20):
            with lo.Descriptor(40, 30, 20, 15, 4, u8, u8) as d:
                setattr(d.desc, field, code)
                pl = C.c_void_p()
                assert L.lancirb200_plan_create(C.c_void_p(d.ptr), C.byref(pl)) == ERR_BAD_ARG, (field, code)
                assert not pl.value
                assert b"element type" in L.avirb200_last_error()


def test_avir_plan_create_refuses_u32():
    rs, v = cs.resizer_and_vars((1, 40, 30, 20, 15, 4, u8, u8, 8, {}))
    h, dp, _ = rs.descriptor((30, 40, 4), u8, 20, 15, u8, 0.0, v)
    try:
        for off in (20, 24):   # avirb200_plan_desc.in_type, .out_type
            field = C.c_int32.from_address(dp + off)
            assert field.value == 0
            field.value = 4
            pl = C.c_void_p()
            assert ab.lib().avirb200_plan_create(C.c_void_p(dp), C.byref(pl)) == ERR_BAD_ARG
            assert not pl.value and b"bad element type" in ab.lib().avirb200_last_error()
            field.value = 0
    finally:
        rs.free_descriptor(h)


def test_avir_host_entry_points_refuse_code_4():
    H = ab.host_lib()
    modes = (C.c_int * 2)()
    for tin, tout in [(4, 0), (0, 4), (4, 4), (-1, 0)]:
        h = H.avirb200_host_desc_create(1, 8, 0, 0, tin, tout, 40, 30, 20, 15, 4, 0.0, 0.0, 0.0, 0, -1, -1, modes)
        assert not h
        assert b"element type" in H.avirb200_host_last_error()
        assert H.avirb200_host_workspace_bytes(1, 8, 0, 0, tin, tout, 40, 30, 20, 15, 4, 0.0, 0.0, 0.0, 0, -1,
                                               -1) == -1
    src = np.zeros((30, 40, 4), u32)
    with pytest.raises(ab.AvirB200Error, match="element type"):
        ab.CImageResizer(8).resizeImage(src, 20, 15)
    with pytest.raises(ab.AvirB200Error, match="element type"):
        ab.CImageResizer(8).resizeImage(np.zeros((30, 40, 4), u8), 20, 15, out_dtype=u32)
    with pytest.raises(ab.AvirB200Error, match="element type"):
        ab.CImageResizer(8).windowFootprint((30, 40, 4), u32, 20, 15, u8, (0, 0, 4, 4))


def test_lancir_host_entry_points_refuse_code_5():
    H = ab.host_lib()
    buf = np.zeros(4096, u8)
    assert H.lancirb200_host_resize(5, 0, buf.ctypes.data, 8, 8, buf.ctypes.data, 4, 4, 1, 0, 0, 0.0, 0.0, 0.0,
                                    0.0, 3.0) == -1
    assert not H.lancirb200_host_desc_create(0, 5, 8, 8, 4, 4, 1, 0.0, 0.0, 0.0, 0.0, 3.0)
    assert not H.lancirb200_host_desc_create(-1, 0, 8, 8, 4, 4, 1, 0.0, 0.0, 0.0, 0.0, 3.0)
    info, nb = (C.c_int * 4)(), C.c_longlong()
    assert H.lancirb200_host_window(2, 0, 5, None, 8, 8, None, 4, 4, 1, 0, 0, 0.0, 0.0, 0.0, 0.0, 3.0, 0, 0, 2, 2,
                                    None, None, info, C.byref(nb)) == -1


@pytest.mark.skipif(ab.device_count() > 0, reason="checks the no-GPU behaviour")
def test_python_clancir_takes_uint32():
    """The Python driver passes uint32 buffers to the library (no GPU: the call returns 0, it does not
    raise)."""
    lr = ab.CLancIR()
    for ti, to in [(u32, u32), (u8, u32), (u32, f32)]:
        r, _ = lr.resizeImage(np.zeros((8, 8, 2), ti), 4, 4, out_dtype=to)
        assert r == 0
        assert lr.windowFootprint((8, 8, 2), ti, 4, 4, to, (0, 0, 2, 2)) is None


@pytest.mark.skipif(ab.device_count() > 0, reason="checks the no-GPU behaviour")
def test_host_c_api_takes_double():
    """double buffers reach the C++ front-end through the host C API (no GPU: CLancIR returns 0)."""
    for ti, to in [(f64, f64), (u8, f64), (f64, u32)]:
        assert lo.front_end(np.zeros((8, 8, 2), ti), 4, 4, to)[0] == 0


def test_python_clancir_rejects_other_dtypes():
    """The Python driver refuses signed, wider and half-precision buffers (and, as before, float64) before the
    library, as source and destination."""
    lr = ab.CLancIR()
    for t in (np.int16, np.int32, np.uint64, np.float16, np.float64):
        with pytest.raises(ab.AvirB200Error, match="uint32 buffers only"):
            lr.resizeImage(np.zeros((8, 8, 4), t), 4, 4)
        with pytest.raises(ab.AvirB200Error, match="uint32 buffers only"):
            lr.resizeImage(np.zeros((8, 8, 4), u8), 4, 4, out_dtype=t)
        with pytest.raises(ab.AvirB200Error, match="uint32 buffers only"):
            lr.resizeImageWindow(np.zeros((8, 8, 4), t), 4, 4, 0, 0, 2, 2)


# ---- the C++ front-end --------------------------------------------------------------------------------------

def build_types_program():
    ab.lib()
    exe = os.path.join(tempfile.mkdtemp(prefix="lancirb200_types_"), "user_types")
    libdir = os.path.join(ROOT, "avir_b200")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "dropin", "user_types.cpp"), "-L" + libdir, "-lavirb200",
                        "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    return exe


@pytest.mark.skipif(ab.device_count() > 0, reason="checks the no-GPU behaviour")
def test_types_program_compiles_and_runs_without_gpu():
    r = subprocess.run([build_types_program()], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert "no device" in r.stdout


def test_other_element_types_do_not_compile(tmp_path):
    src = tmp_path / "int16.cpp"
    src.write_text('#include "lancir_b200.h"\n'
                   "int main() {\n"
                   "    static int16_t in[16], out[4];\n"
                   "    avir::CLancIR L;\n"
                   "    return L.resizeImage(in, 4, 4, out, 2, 2, 1);\n"
                   "}\n")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode != 0
    assert "CLancIR element types are uint8_t, uint16_t, float, double and uint32_t" in r.stderr
