"""ctypes mirror of the C++ front-end API (same names and argument meaning as upstream).

``CImageResizer(res_bits, src_bits, params, fpclass).resizeImage(src, NewWidth, NewHeight, k,
vars)`` drives ``avir::CImageResizer<fpclass>::resizeImage`` of ``include/avir_b200.h``
through ``libavirb200_host.so``; ``resizeImageDevice`` takes CUDA device pointers (e.g. from
torch tensors).  Arrays are numpy, shaped (H, W, C), dtype uint8 / uint16 / float32 / float64 (CImageResizer)
or uint8 / uint16 / float32 / uint32 (CLancIR; upstream lancir.h treats uint32 as uint16).
"""
import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))

FP_DEF, FP_FLOAT4, FP_FLOAT8_DIL = 0, 1, 2
# the same classes composed with upstream's error-diffusion ditherer (CImageResizerDithererErrdINL/DIL)
FP_DEF_ERRD, FP_FLOAT4_ERRD, FP_FLOAT8_DIL_ERRD = 3, 4, 5
_T = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float32): 2, np.dtype(np.float64): 3,
      np.dtype(np.uint32): 4}


# avirb200_plan_set_option() keys (include/avirb200.h, avirb200_option)
OPT_KERNEL_FAMILY, OPT_STREAM_VARIANT_H, OPT_STREAM_VARIANT_V, OPT_HOST_BANDS, OPT_ALL_STREAM_CHAINS, OPT_OVERLAP_HALO = range(6)


class AvirB200Error(RuntimeError):
    pass


# CLancIR buffer types of this driver; CImageResizer refuses uint32 (code 4) with AvirB200Error.  double
# CLancIR buffers are the C++ front-end's (lancir_b200.h; lancirb200_host_resize / _window with code 3).
_LT = (np.dtype(np.uint8), np.dtype(np.uint16), np.dtype(np.float32), np.dtype(np.uint32))


_lib = None
_host = None


def lib():
    """libavirb200.so (C ABI, include/avirb200.h)."""
    global _lib
    if _lib is None:
        path = os.path.join(_PKG, "libavirb200.so")
        if not os.path.exists(path):
            raise AvirB200Error("libavirb200.so is not built: run `python avir_b200/build.py` "
                                "(there is no CPU fallback)")
        _lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
        _lib.avirb200_status_string.restype = C.c_char_p
        _lib.avirb200_last_error.restype = C.c_char_p
    return _lib


def host_lib():
    """libavirb200_host.so (the C++ front-ends behind a C API)."""
    global _host
    if _host is None:
        lib()
        path = os.path.join(_PKG, "libavirb200_host.so")
        if not os.path.exists(path):
            raise AvirB200Error("libavirb200_host.so is not built: run `python avir_b200/build.py`")
        h = C.CDLL(path)
        h.avirb200_host_last_error.restype = C.c_char_p
        h.avirb200_host_set_option.argtypes = [C.c_int, C.c_int]
        call = [C.c_int] * 6
        geom = [C.c_int] * 5 + [C.c_double] * 3 + [C.c_int] * 3
        h.avirb200_host_desc_create.restype = C.c_void_p
        h.avirb200_host_desc_create.argtypes = call + geom + [C.c_void_p]
        h.avirb200_host_desc_get.restype = C.c_void_p
        h.avirb200_host_desc_get.argtypes = [C.c_void_p]
        h.avirb200_host_desc_free.argtypes = [C.c_void_p]
        h.avirb200_host_resize.restype = C.c_int
        h.avirb200_host_resize.argtypes = call + [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                  C.c_int, C.c_int, C.c_int] + [C.c_double] * 3 + [
                                                      C.c_int] * 3
        h.avirb200_host_resize_device.restype = C.c_int
        h.avirb200_host_resize_device.argtypes = h.avirb200_host_resize.argtypes + [C.c_void_p,
                                                                                    C.c_void_p]
        h.avirb200_host_workspace_bytes.restype = C.c_longlong
        h.avirb200_host_workspace_bytes.argtypes = call + geom
        h.avirb200_host_window.restype = C.c_int
        h.avirb200_host_window.argtypes = ([C.c_int] + h.avirb200_host_resize.argtypes + [C.c_int] * 4 +
                                           [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p])
        h.lancirb200_host_resize.restype = C.c_int
        h.lancirb200_host_resize.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                             C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                             C.c_double, C.c_double, C.c_double, C.c_double,
                                             C.c_double]
        h.lancirb200_host_desc_create.restype = C.c_void_p
        h.lancirb200_host_desc_create.argtypes = [C.c_int] * 7 + [C.c_double] * 5
        h.lancirb200_host_desc_get.restype = C.c_void_p
        h.lancirb200_host_desc_get.argtypes = [C.c_void_p]
        h.lancirb200_host_desc_free.argtypes = [C.c_void_p]
        h.lancirb200_host_window.restype = C.c_int
        h.lancirb200_host_window.argtypes = ([C.c_int] + h.lancirb200_host_resize.argtypes + [C.c_int] * 4 +
                                             [C.c_void_p] * 4)
        _host = h
    return _host


def device_count():
    return lib().avirb200_device_count()


def set_option(option, value):
    """Test / tuning hook of the ctypes driver: plan option applied to every plan the front-end
    objects behind host_lib() use from now on (value -1: back to the plan's default)."""
    host_lib().avirb200_host_set_option(option, value)


def _scanlines(buf, pitch, what):
    """Pointer to an (H, W, C) image whose rows lie `pitch` elements apart (pitch < 1: packed rows).
    With a pitch the caller's array is used as it is -- typically a strided view into a larger,
    padded backing array -- so its pixels must be packed within each row."""
    if pitch < 1:
        return np.ascontiguousarray(buf)
    it = buf.dtype.itemsize
    h, w, c = buf.shape
    if buf.strides[1:] != (c * it, it) or (h > 1 and buf.strides[0] != pitch * it) or pitch < w * c:
        raise AvirB200Error("%s: an (H, W, C) view with packed pixels and rows %d elements apart is "
                            "needed for a scanline size of %d" % (what, pitch, pitch))
    return buf


class CImageResizerVars:
    """Upstream avir.h:2516-2547 (input members)."""

    def __init__(self, ox=0.0, oy=0.0, UseSRGBGamma=False, AlphaIndex=-1, BuildMode=-1):
        self.ox, self.oy = ox, oy
        self.UseSRGBGamma, self.AlphaIndex, self.BuildMode = UseSRGBGamma, AlphaIndex, BuildMode


class CImageResizer:
    """avir::CImageResizer<fpclass>(aResBitDepth, aSrcBitDepth, aParams), avir.h:4630."""

    def __init__(self, aResBitDepth=8, aSrcBitDepth=0, aParams=0, fpclass=FP_DEF):
        self.res_bits, self.src_bits, self.params, self.fpclass = (aResBitDepth, aSrcBitDepth,
                                                                  aParams, fpclass)

    def _call(self, tin, tout):
        return (self.fpclass, self.res_bits, self.src_bits, self.params, tin, tout)

    @staticmethod
    def _vars(v):
        v = v or CImageResizerVars()
        return v.ox, v.oy, int(v.UseSRGBGamma), v.AlphaIndex, v.BuildMode

    def resizeImage(self, SrcBuf, NewWidth, NewHeight, k=0.0, aVars=None, out_dtype=None,
                    NewBuf=None, SrcScanlineSize=0):
        """Host buffers in, host buffers out (avir.h:4680-4685).  SrcScanlineSize > 0: SrcBuf's
        rows lie that many elements apart (SrcBuf a strided view into the padded buffer)."""
        src = _scanlines(SrcBuf, SrcScanlineSize, "resizeImage")
        sh, sw, ch = src.shape
        out_dtype = np.dtype(out_dtype or src.dtype)
        dst = NewBuf if NewBuf is not None else np.empty((NewHeight, NewWidth, ch), out_dtype)
        ox, oy, g, a, bm = self._vars(aVars)
        r = host_lib().avirb200_host_resize(*self._call(_T[src.dtype], _T[out_dtype]),
                                            src.ctypes.data, sw, sh, SrcScanlineSize,
                                            dst.ctypes.data, NewWidth, NewHeight, ch, k, ox, oy, g,
                                            a, bm)
        if r != 0:
            raise AvirB200Error(host_lib().avirb200_host_last_error().decode())
        return dst

    def workspaceBytes(self, src_shape, in_dtype, NewWidth, NewHeight, out_dtype, k=0.0, aVars=None):
        sh, sw, ch = src_shape
        ox, oy, g, a, bm = self._vars(aVars)
        n = host_lib().avirb200_host_workspace_bytes(
            *self._call(_T[np.dtype(in_dtype)], _T[np.dtype(out_dtype)]), sw, sh, NewWidth,
            NewHeight, ch, k, ox, oy, g, a, bm)
        if n < 0:
            raise AvirB200Error(host_lib().avirb200_host_last_error().decode())
        return int(n)

    def resizeImageDevice(self, d_src, src_shape, in_dtype, d_dst, NewWidth, NewHeight, out_dtype,
                          d_workspace, k=0.0, aVars=None, stream=0, SrcScanlineSize=0):
        """Device pointers (ints); asynchronous on `stream` (GPU extension).  SrcScanlineSize:
        elements from one source row to the next (< 1: packed rows)."""
        sh, sw, ch = src_shape
        ox, oy, g, a, bm = self._vars(aVars)
        r = host_lib().avirb200_host_resize_device(
            *self._call(_T[np.dtype(in_dtype)], _T[np.dtype(out_dtype)]), d_src, sw, sh,
            SrcScanlineSize, d_dst,
            NewWidth, NewHeight, ch, k, ox, oy, g, a, bm, d_workspace, stream)
        if r != 0:
            raise AvirB200Error(host_lib().avirb200_host_last_error().decode())

    def _window(self, op, src, src_shape, in_dtype, src_pitch, dst, NewWidth, NewHeight, out_dtype, k, aVars,
                window, d_workspace=None, stream=0):
        sh, sw, ch = src_shape
        ox, oy, g, a, bm = self._vars(aVars)
        info, nbytes = (C.c_int * 6)(), C.c_longlong(0)
        r = host_lib().avirb200_host_window(op, *self._call(_T[np.dtype(in_dtype)], _T[np.dtype(out_dtype)]), src, sw,
                                            sh, src_pitch, dst, NewWidth, NewHeight, ch, k, ox, oy, g, a, bm,
                                            *window, d_workspace, stream, info, C.byref(nbytes))
        if r != 0:
            raise AvirB200Error(host_lib().avirb200_host_last_error().decode())
        return list(info), nbytes.value

    def resizeImageWindow(self, SrcBuf, NewWidth, NewHeight, window, k=0.0, aVars=None, out_dtype=None,
                          NewBuf=None, SrcScanlineSize=0):
        """The destination window (x0, y0, w, h) of resizeImage(SrcBuf, NewWidth, NewHeight, ...):
        SrcBuf is the whole source (host), the result is an (h, w, C) array (GPU extension)."""
        src = _scanlines(SrcBuf, SrcScanlineSize, "resizeImageWindow")
        out_dtype = np.dtype(out_dtype or src.dtype)
        dst = NewBuf if NewBuf is not None else np.empty((window[3], window[2], src.shape[2]), out_dtype)
        self._window(0, src.ctypes.data, src.shape, src.dtype, SrcScanlineSize, dst.ctypes.data, NewWidth,
                     NewHeight, out_dtype, k, aVars, window)
        return dst

    def resizeImageWindowDevice(self, d_src, src_shape, in_dtype, d_dst, NewWidth, NewHeight, out_dtype, window,
                                d_workspace, k=0.0, aVars=None, stream=0, SrcScanlineSize=0):
        """Device pointers: d_src at the window's footprint (windowFootprint), d_dst receives the (h, w, C)
        window; src_shape is the WHOLE source's (H, W, C).  Asynchronous on `stream`."""
        self._window(1, d_src, src_shape, in_dtype, SrcScanlineSize, d_dst, NewWidth, NewHeight, out_dtype, k, aVars,
                     window, d_workspace, stream)

    def windowFootprint(self, src_shape, in_dtype, NewWidth, NewHeight, out_dtype, window, k=0.0, aVars=None):
        """dict of avirb200_window_info: the source columns / rows the window reads."""
        info, _ = self._window(2, None, src_shape, in_dtype, 0, None, NewWidth, NewHeight, out_dtype, k, aVars,
                               window)
        return dict(zip(("src_x0", "src_w", "src_y0", "src_h", "mid_row0", "mid_rows"), info))

    def windowWorkspaceBytes(self, src_shape, in_dtype, NewWidth, NewHeight, out_dtype, window, k=0.0, aVars=None):
        return self._window(3, None, src_shape, in_dtype, 0, None, NewWidth, NewHeight, out_dtype, k, aVars,
                            window)[1]

    def descriptor(self, src_shape, in_dtype, NewWidth, NewHeight, out_dtype, k=0.0, aVars=None):
        """Host-only: the C-ABI plan descriptor resizeImage would hand to the GPU library.
        Returns (handle, desc_ptr, (mode_h, mode_v)); free with free_descriptor(handle)."""
        sh, sw, ch = src_shape
        ox, oy, g, a, bm = self._vars(aVars)
        modes = (C.c_int * 2)()
        h = host_lib().avirb200_host_desc_create(
            *self._call(_T[np.dtype(in_dtype)], _T[np.dtype(out_dtype)]), sw, sh, NewWidth,
            NewHeight, ch, k, ox, oy, g, a, bm, modes)
        if not h:
            raise AvirB200Error(host_lib().avirb200_host_last_error().decode())
        return h, host_lib().avirb200_host_desc_get(h), (modes[0], modes[1])

    @staticmethod
    def free_descriptor(handle):
        host_lib().avirb200_host_desc_free(handle)


class CLancIRParams:
    """Upstream lancir.h:260-307."""

    def __init__(self, SrcSSize=0, NewSSize=0, kx=0.0, ky=0.0, ox=0.0, oy=0.0, la=3.0):
        self.SrcSSize, self.NewSSize, self.kx, self.ky, self.ox, self.oy, self.la = (
            SrcSSize, NewSSize, kx, ky, ox, oy, la)


class CLancIR:
    """avir::CLancIR, lancir.h:311 (1-4 channel images, u8 / u16 / float / uint32 buffers)."""

    def resizeImage(self, SrcBuf, NewWidth, NewHeight, aParams=None, out_dtype=None, NewBuf=None):
        """aParams.SrcSSize / NewSSize > 0: SrcBuf / NewBuf are (H, W, C) views whose rows lie that
        many elements apart (strided views into padded buffers; NewBuf is then required)."""
        p = aParams or CLancIRParams()
        src = _scanlines(SrcBuf, p.SrcSSize, "CLancIR.resizeImage (SrcSSize)")
        sh, sw, ch = src.shape
        out_dtype = np.dtype(out_dtype or (NewBuf.dtype if NewBuf is not None else src.dtype))
        if NewBuf is None:
            if p.NewSSize > 0:
                raise AvirB200Error("CLancIR.resizeImage: NewSSize needs a caller-supplied NewBuf")
            dst = np.empty((NewHeight, NewWidth, ch), out_dtype)
        else:
            dst = NewBuf
            if dst.shape != (NewHeight, NewWidth, ch) or dst.dtype != out_dtype:
                raise AvirB200Error("CLancIR.resizeImage: NewBuf is not (NewHeight, NewWidth, C) of out_dtype")
            if p.NewSSize > 0:
                _scanlines(dst, p.NewSSize, "CLancIR.resizeImage (NewSSize)")
            elif not dst.flags.c_contiguous:
                raise AvirB200Error("CLancIR.resizeImage: NewBuf must be contiguous without NewSSize")
        if src.dtype not in _LT or out_dtype not in _LT:
            raise AvirB200Error("CLancIR: uint8 / uint16 / float32 / uint32 buffers only")
        r = host_lib().lancirb200_host_resize(_T[src.dtype], _T[out_dtype], src.ctypes.data, sw, sh,
                                              dst.ctypes.data, NewWidth, NewHeight, ch, p.SrcSSize,
                                              p.NewSSize, p.kx, p.ky, p.ox, p.oy, p.la)
        return r, dst

    @staticmethod
    def _window(op, src, src_shape, in_dtype, dst, NewWidth, NewHeight, out_dtype, win, p, d_workspace=None,
                stream=0):
        sh, sw, ch = src_shape
        in_dtype, out_dtype = np.dtype(in_dtype), np.dtype(out_dtype)
        if in_dtype not in _LT or out_dtype not in _LT:
            raise AvirB200Error("CLancIR: uint8 / uint16 / float32 / uint32 buffers only")
        info, nbytes = (C.c_int * 4)(), C.c_longlong(0)
        r = host_lib().lancirb200_host_window(op, _T[in_dtype], _T[out_dtype], src, sw, sh, dst, NewWidth, NewHeight,
                                              ch, p.SrcSSize, p.NewSSize, p.kx, p.ky, p.ox, p.oy, p.la, *win,
                                              d_workspace, stream, info, C.byref(nbytes))
        return r, list(info), nbytes.value

    def resizeImageWindow(self, SrcBuf, NewWidth, NewHeight, WinX, WinY, WinWidth, WinHeight, aParams=None,
                          out_dtype=None, NewBuf=None):
        """The destination window (WinX, WinY, WinWidth, WinHeight) of resizeImage(SrcBuf, NewWidth, NewHeight,
        aParams) (GPU extension): SrcBuf is the whole source, the result an (WinHeight, WinWidth, C) array.
        aParams.SrcSSize / NewSSize as in resizeImage (NewSSize: the window's scanline size).  Returns
        (WinHeight or 0, window)."""
        p = aParams or CLancIRParams()
        src = _scanlines(SrcBuf, p.SrcSSize, "CLancIR.resizeImageWindow (SrcSSize)")
        ch = src.shape[2]
        out_dtype = np.dtype(out_dtype or (NewBuf.dtype if NewBuf is not None else src.dtype))
        shape = (max(WinHeight, 0), max(WinWidth, 0), ch)
        if NewBuf is None:
            if p.NewSSize > 0:
                raise AvirB200Error("CLancIR.resizeImageWindow: NewSSize needs a caller-supplied NewBuf")
            dst = np.empty(shape, out_dtype)
        else:
            dst = NewBuf
            if dst.shape != shape or dst.dtype != out_dtype:
                raise AvirB200Error("CLancIR.resizeImageWindow: NewBuf is not (WinHeight, WinWidth, C) of out_dtype")
            if p.NewSSize > 0:
                _scanlines(dst, p.NewSSize, "CLancIR.resizeImageWindow (NewSSize)")
            elif not dst.flags.c_contiguous:
                raise AvirB200Error("CLancIR.resizeImageWindow: NewBuf must be contiguous without NewSSize")
        r, _, _ = self._window(0, src.ctypes.data, src.shape, src.dtype, dst.ctypes.data, NewWidth, NewHeight,
                               out_dtype, (WinX, WinY, WinWidth, WinHeight), p)
        return r, dst

    def resizeImageWindowDevice(self, d_src, src_shape, in_dtype, d_dst, NewWidth, NewHeight, out_dtype, window,
                                d_workspace, aParams=None, stream=0):
        """Device pointers: d_src at the window's footprint (windowFootprint), d_dst receives the window;
        src_shape is the WHOLE source's (H, W, C).  Asynchronous on `stream`.  Returns WinHeight or 0."""
        return self._window(1, d_src, src_shape, in_dtype, d_dst, NewWidth, NewHeight, out_dtype, window,
                            aParams or CLancIRParams(), d_workspace, stream)[0]

    def windowFootprint(self, src_shape, in_dtype, NewWidth, NewHeight, out_dtype, window, aParams=None):
        """dict of lancirb200_window_info (the source columns / rows the window reads), None where the
        front-end returns 0."""
        r, info, _ = self._window(2, None, src_shape, in_dtype, None, NewWidth, NewHeight, out_dtype, window,
                                  aParams or CLancIRParams())
        return dict(zip(("src_x0", "src_w", "src_y0", "src_h"), info)) if r > 0 else None

    def windowWorkspaceBytes(self, src_shape, in_dtype, NewWidth, NewHeight, out_dtype, window, aParams=None):
        """Device workspace bytes of resizeImageWindowDevice (0 where the front-end returns 0)."""
        return self._window(3, None, src_shape, in_dtype, None, NewWidth, NewHeight, out_dtype, window,
                            aParams or CLancIRParams())[2]
