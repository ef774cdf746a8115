"""CLancIR with every element type upstream lists (uint8_t, uint16_t, float, double, uint32_t): access to the
oracles and to the C++ front-end for tests/test_lancir_types.py and tests/test_gpu_lancir_types.py
(TEST INFRASTRUCTURE).

* ``oracle/_ref/liblancir_types_ref.so`` -- upstream's lancir.h, unmodified, through
  ``oracle/lancir_types_shim.cpp`` with the pinned flags (``oracle/types.mk``);
* ``oracle/liblancir_types_port.so`` -- the C port's CLancIR with every type's load and output stage
  (``oracle/lancir_types_port.c``);
* the C++ front-end ``avir::CLancIR`` through the host C API (``lancirb200_host_resize`` /
  ``lancirb200_host_window``), which takes all five types;
* descriptors and device plans of a call, as ``CLancIR::resizeImage`` builds them.
"""
import contextlib
import ctypes as C
import os

import numpy as np

import avir_b200 as ab
from test_lancir_window import LancirDesc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, "oracle", "_ref", "liblancir_types_ref.so")
PORT_SO = os.path.join(ROOT, "oracle", "liblancir_types_port.so")

# avirb200_dtype codes
CODE = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float32): 2, np.dtype(np.float64): 3,
        np.dtype(np.uint32): 4}

_ref = None
_port = None


def code(t):
    return CODE[np.dtype(t)]


def have_ref():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        lib = C.CDLL(REF_SO)
        lib.lancir_types_ref_resize.restype = C.c_int
        lib.lancir_types_ref_resize.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int,
                                                C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_double] * 5
        _ref = lib
    return _ref


def port():
    global _port
    if _port is None:
        lib = C.CDLL(PORT_SO)
        lib.lancir_types_port_resize.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
        lib.lancir_types_port_resize.restype = C.c_int
        _port = lib
    return _port


def _rows(a, pitch):
    """a itself when its rows lie `pitch` elements apart with packed pixels, a contiguous copy when pitch < 1."""
    if pitch < 1:
        return np.ascontiguousarray(a)
    it = a.dtype.itemsize
    assert a.strides[1:] == (a.shape[2] * it, it) and (a.shape[0] < 2 or a.strides[0] == pitch * it)
    return a


def _kw(kw):
    kw = kw or {}
    return kw.get("kx", 0.0), kw.get("ky", 0.0), kw.get("ox", 0.0), kw.get("oy", 0.0), kw.get("la", 3.0)


def lancir_ref(src, nw, nh, out_dtype, kw=None, srcssize=0, newssize=0, dst=None):
    """Upstream CLancIR::resizeImage: (return value, destination).  srcssize / newssize > 0: src / dst are
    strided views into padded buffers (dst, required with newssize, is written in place)."""
    src = _rows(src, srcssize)
    sh, sw, c = src.shape
    if dst is None:
        assert newssize < 1
        dst = np.zeros((nh, nw, c), dtype=out_dtype)
    else:
        dst = _rows(dst, newssize)
    r = ref().lancir_types_ref_resize(code(src.dtype), code(out_dtype), src.ctypes.data, sw, sh, dst.ctypes.data,
                                      nw, nh, c, srcssize, newssize, *_kw(kw))
    return r, dst


class Descriptor:
    """The descriptor CLancIR::resizeImage builds for the call (host only)."""

    def __init__(self, sw, sh, nw, nh, ch, ti, to, kw=None):
        self.handle = ab.host_lib().lancirb200_host_desc_create(code(ti), code(to), sw, sh, nw, nh, ch, *_kw(kw))
        assert self.handle
        self.ptr = ab.host_lib().lancirb200_host_desc_get(self.handle)
        self.desc = LancirDesc.from_address(self.ptr)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        ab.host_lib().lancirb200_host_desc_free(self.handle)


def port_resize(src, nw, nh, to, kw=None):
    """The C port on the descriptor CLancIR::resizeImage builds for the call."""
    sh, sw, ch = src.shape
    src = np.ascontiguousarray(src)
    with Descriptor(sw, sh, nw, nh, ch, src.dtype, to, kw) as d:
        dst = np.zeros((nh, nw, ch), to)
        assert port().lancir_types_port_resize(d.ptr, src.ctypes.data, sw * ch, dst.ctypes.data, nw * ch) == 0
    return dst


def expected(src, nw, nh, to, kw=None):
    """Upstream's output, or the C port's where oracle/_ref is absent."""
    if have_ref():
        r, want = lancir_ref(src, nw, nh, to, kw)
        assert r == nh
        return want
    return port_resize(src, nw, nh, to, kw)


def front_end(src, nw, nh, to, kw=None, srcssize=0, newssize=0, dst=None):
    """avir::CLancIR::resizeImage (lancir_b200.h) with host buffers: (return value, destination); srcssize /
    newssize as in lancir_ref."""
    src = _rows(src, srcssize)
    sh, sw, ch = src.shape
    if dst is None:
        assert newssize < 1
        dst = np.zeros((nh, nw, ch), to)
    else:
        dst = _rows(dst, newssize)
    r = ab.host_lib().lancirb200_host_resize(code(src.dtype), code(to), src.ctypes.data, sw, sh, dst.ctypes.data, nw,
                                             nh, ch, srcssize, newssize, *_kw(kw))
    return r, dst


def front_end_window(src, nw, nh, to, win, kw=None):
    """avir::CLancIR::resizeImageWindow with host buffers: (return value, the (h, w, C) window)."""
    src = np.ascontiguousarray(src)
    sh, sw, ch = src.shape
    dst = np.zeros((win[3], win[2], ch), to)
    info, nb = (C.c_int * 4)(), C.c_longlong()
    r = ab.host_lib().lancirb200_host_window(0, code(src.dtype), code(to), src.ctypes.data, sw, sh, dst.ctypes.data,
                                             nw, nh, ch, 0, 0, *_kw(kw), *win, None, None, info, C.byref(nb))
    return r, dst


@contextlib.contextmanager
def lancir_plan(sw, sh, nw, nh, ch, ti, to, kw=None):
    """A C-ABI plan of the call, as CLancIR::resizeImage builds it; yields (library, plan, descriptor)."""
    from test_gpu_lancir_window import llib
    with Descriptor(sw, sh, nw, nh, ch, ti, to, kw) as d:
        L, pl = llib(), C.c_void_p()
        try:
            r = L.lancirb200_plan_create(C.c_void_p(d.ptr), C.byref(pl))
            assert r == 0, L.avirb200_last_error().decode()
            yield L, pl, d.ptr
        finally:
            if pl.value:
                L.lancirb200_plan_destroy(pl)
