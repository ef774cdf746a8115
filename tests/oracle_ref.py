"""ctypes access to the parity oracles (TEST INFRASTRUCTURE).

* ``oracle/_ref/libavir_ref.so`` -- the unmodified upstream headers compiled through
  ``oracle/ref_shim.cpp`` (pinned flags ``-O2 -mavx2 -ffp-contract=off``).
* helpers shared by the tests: the SURVEY.md section 8(d) xorshift32 input generator and the
  FNV-1a-64 hash used by the App. A smoke KATs.

Nothing in the product package imports this module.
"""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libavir_ref.so")

FP_DEF, FP_FLOAT4, FP_FLOAT8_DIL = 0, 1, 2
T_U8, T_U16, T_F32 = 0, 1, 2
NP_T = {T_U8: np.uint8, T_U16: np.uint16, T_F32: np.float32}
T_OF = {np.dtype(np.uint8): T_U8, np.dtype(np.uint16): T_U16, np.dtype(np.float32): T_F32,
        np.dtype(np.float64): 3}

_ref = None


def have_ref():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_SO)
        lib.avir_ref_resize.restype = C.c_int
        lib.avir_ref_resize.argtypes = [
            C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
            C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_double, C.c_double,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
        lib.avir_ref_plan.restype = C.c_long
        lib.avir_ref_plan.argtypes = [
            C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
            C.c_int, C.c_int, C.c_int, C.c_double, C.c_int, C.c_int, C.c_double, C.c_double,
            C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_long]
        lib.lancir_ref_resize.restype = C.c_int
        lib.lancir_ref_resize.argtypes = [
            C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
            C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double,
            C.c_double]
        lib.avir_ref_version.restype = C.c_char_p
        _ref = lib
    return _ref


def xorshift32_image(h, w, c, dtype, seed=12345):
    """SURVEY.md 8(d): one xorshift32 draw per element in memory order,
    element = (T)((draw & 0xFFFF) * scale), scale 1 (u16), 1/257 (u8), 1/65535 (f32)."""
    n = h * w * c
    out = np.empty(n, dtype=np.uint32)
    x = np.uint32(seed)
    # vectorising xorshift is awkward; do it in chunks with python ints (fast enough
    # for test sizes) -- large images use xorshift32_image_fast().
    s = int(seed)
    buf = out
    for i in range(n):
        s ^= (s << 13) & 0xFFFFFFFF
        s ^= s >> 17
        s ^= (s << 5) & 0xFFFFFFFF
        buf[i] = s
    return _scale_draws(out, dtype).reshape(h, w, c)


def _scale_draws(draws, dtype):
    lo = (draws & 0xFFFF).astype(np.float64)
    dtype = np.dtype(dtype)
    if dtype == np.uint16:
        return lo.astype(np.uint16)
    if dtype == np.uint8:
        return (lo * (1.0 / 257)).astype(np.uint8)
    if dtype == np.float64:
        return lo * (1.0 / 65535)  # not representable in float: the (float) cast of the path rounds
    return (lo * (1.0 / 65535)).astype(np.float32)


def lcg_image(h, w, c, dtype, seed=1):
    """Fast vectorised pseudo-random image for larger parity cases (not a KAT input)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    draws = rng.integers(0, 1 << 32, size=h * w * c, dtype=np.uint32)
    return _scale_draws(draws, dtype).reshape(h, w, c)


def fnv1a64(a):
    hsh = 0xcbf29ce484222325
    for b in np.ascontiguousarray(a).view(np.uint8).ravel().tolist():
        hsh ^= b
        hsh = (hsh * 0x100000001b3) & 0xFFFFFFFFFFFFFFFF
    return "%016x" % hsh


def _rows(a, pitch):
    """a itself when its rows lie `pitch` elements apart with packed pixels (a strided view into a
    padded buffer: upstream then reads that buffer), a contiguous copy when pitch < 1."""
    if pitch < 1:
        return np.ascontiguousarray(a)
    it = a.dtype.itemsize
    assert a.strides[1:] == (a.shape[2] * it, it) and (a.shape[0] < 2 or a.strides[0] == pitch * it)
    return a


def ref_resize(src, nw, nh, out_dtype, fpclass=FP_FLOAT4, k=0.0, resbits=8, srcbits=0,
               ox=0.0, oy=0.0, gamma=False, alpha=-1, buildmode=-1, nthreads=1, params=0,
               src_pitch=0):
    """Upstream resizeImage; src_pitch > 0 is its SrcScanlineSize (src a strided view, see _rows)."""
    src = _rows(src, src_pitch)
    sh, sw, c = src.shape
    dst = np.zeros((nh, nw, c), dtype=out_dtype)
    r = ref().avir_ref_resize(fpclass, T_OF[src.dtype], T_OF[np.dtype(out_dtype)],
                              src.ctypes.data, sw, sh, src_pitch, dst.ctypes.data, nw, nh, c,
                              k, resbits, srcbits, ox, oy, int(gamma), alpha, buildmode,
                              nthreads, params)
    assert r == 0
    return dst


def ref_plan(src, nw, nh, out_dtype, fpclass=FP_FLOAT4, k=0.0, resbits=8, srcbits=0,
             ox=0.0, oy=0.0, gamma=False, alpha=-1, buildmode=-1, params=0):
    """Plan that upstream resizeImage() built, as {'H': [steps], 'V': [steps]}."""
    src = np.ascontiguousarray(src)
    sh, sw, c = src.shape
    dst = np.zeros((nh, nw, c), dtype=out_dtype)
    args = (fpclass, T_OF[src.dtype], T_OF[np.dtype(out_dtype)], src.ctypes.data, sw, sh, 0,
            dst.ctypes.data, nw, nh, c, k, resbits, srcbits, ox, oy, int(gamma), alpha,
            buildmode, params)
    n = ref().avir_ref_plan(*args, None, 0)
    assert n > 0
    buf = np.zeros(n, dtype=np.float64)
    n2 = ref().avir_ref_plan(*args, buf.ctypes.data, n)
    assert n2 == n
    return parse_plan(buf), dst


def parse_plan(buf):
    pos = [0]

    def take(n=1):
        v = buf[pos[0]:pos[0] + n]
        pos[0] += n
        return v

    plan = {}
    for name in ("H", "V"):
        steps = []
        ns = int(take()[0])
        for _ in range(ns):
            hd = take(11).astype(np.int64)
            s = dict(zip(["kind", "R", "lat", "edge", "InLen", "InPrefix", "InSuffix", "OutLen",
                          "OutPrefix", "OutSuffix", "FltOrigLen"], [int(v) for v in hd]))
            nf = int(take()[0])
            s["Flt"] = take(nf).astype(np.float32)
            s["FL"], s["order"], s["FracCount"], npos = [int(v) for v in take(4)]
            p = take(npos * 4).reshape(npos, 4)
            s["SrcPosInt"] = p[:, 0].astype(np.int32)
            s["fti"] = p[:, 1].astype(np.int32)
            s["x"] = p[:, 2].astype(np.float32)
            s["fl"] = p[:, 3].astype(np.int32)
            nu = int(take()[0])
            fs = s["FL"] * (s["order"] + 1)
            s["bank"] = {}
            for _u in range(nu):
                f = int(take()[0])
                s["bank"][f] = take(fs).astype(np.float32)
            steps.append(s)
        plan[name] = steps
    assert pos[0] == len(buf)
    return plan


def lancir_ref(src, nw, nh, out_dtype, kx=0.0, ky=0.0, ox=0.0, oy=0.0, la=3.0, srcssize=0,
               newssize=0, dst=None):
    """Upstream CLancIR::resizeImage.  srcssize / newssize > 0 are its SrcSSize / NewSSize: src /
    dst are then strided views into padded buffers (dst, required with newssize, is written in
    place and returned)."""
    src = _rows(src, srcssize)
    sh, sw, c = src.shape
    if dst is None:
        assert newssize < 1
        dst = np.zeros((nh, nw, c), dtype=out_dtype)
    else:
        dst = _rows(dst, newssize)
        assert dst.shape == (nh, nw, c) and dst.dtype == np.dtype(out_dtype)
    r = ref().lancir_ref_resize(T_OF[src.dtype], T_OF[np.dtype(out_dtype)], src.ctypes.data,
                                sw, sh, dst.ctypes.data, nw, nh, c, srcssize, newssize, kx, ky, ox,
                                oy, la)
    return r, dst
