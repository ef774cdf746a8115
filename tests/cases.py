"""Shared parity cases and helpers.

A case is (fpclass, src_w, src_h, new_w, new_h, channels, in_dtype, out_dtype, res_bits, kwargs)
with kwargs drawn from: gamma, alpha, buildmode, ox, oy, k, params.
"""
import ctypes as C
import os

import numpy as np

import avir_b200 as ab
import oracle_ref as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64

# Scaled-down versions of the BASELINE.json configs first, then coverage of every chain
# shape, type combination, channel count and option (SURVEY.md section 8f rank 4).
SMALL_CASES = [
    # cfg2: 2X upsize u8 RGBA (k = 0.5); auto mode on small images picks filtered upsample
    (1, 240, 135, 480, 270, 4, u8, u8, 8, {}),
    (1, 240, 135, 480, 270, 4, u8, u8, 8, {"buildmode": 1}),   # the chain big images select
    # cfg3: 8K->4K float RGBA (k = 2), both mirrors named by the north star
    (2, 192, 108, 96, 54, 4, f32, f32, 16, {}),
    (2, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1}),
    (1, 192, 108, 96, 54, 4, f32, f32, 16, {}),
    (1, 192, 108, 96, 54, 4, f32, f32, 16, {"buildmode": 1}),
    # cfg4: 4X downsize u16 RGBA (k = 4), decimating FIR
    (1, 256, 256, 64, 64, 4, u16, u16, 16, {}),
    (1, 256, 256, 64, 64, 4, u16, u16, 16, {"buildmode": 1}),
    # cfg5: planar/DIL mirror, 4X downsize u8 + sRGB gamma, alpha exempt
    (2, 384, 216, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),
    (2, 384, 216, 96, 54, 4, u8, u8, 8, {"gamma": True, "alpha": 3, "buildmode": 1}),
    # cfg1 geometry through AVIR (k = 0.625), default class, RGB
    (0, 64, 48, 100, 75, 3, u8, u8, 8, {}),
    (1, 64, 48, 100, 75, 4, u8, u8, 8, {}),
    (2, 64, 48, 100, 75, 4, u8, u8, 8, {}),
    (2, 64, 48, 100, 75, 4, u8, u8, 8, {"buildmode": 1}),
    # 1 < k < 2, non-integer ratios, kx != ky
    (1, 100, 60, 67, 41, 2, u16, u16, 16, {}),
    (2, 150, 90, 100, 55, 4, f32, f32, 16, {"buildmode": 1}),
    (0, 150, 90, 100, 55, 3, u8, u8, 8, {"buildmode": 1}),
    (1, 100, 60, 150, 77, 4, u8, u8, 8, {}),
    (2, 100, 60, 150, 77, 4, u8, u8, 8, {}),
    # large ratios
    (2, 200, 120, 25, 15, 4, u16, u16, 16, {}),
    (0, 400, 240, 25, 15, 1, u8, u8, 8, {}),
    (1, 333, 211, 40, 27, 4, f32, f32, 16, {"buildmode": 0}),
    # mixed types / OutMul != 1 / gamma variants / float-out quirk of the default class
    (1, 300, 200, 200, 133, 4, u8, u16, 16, {}),
    (1, 120, 80, 60, 40, 4, u16, u8, 16, {}),
    (1, 120, 80, 60, 40, 4, f32, u8, 8, {}),
    (1, 120, 80, 60, 40, 4, u8, f32, 8, {}),
    (1, 192, 108, 48, 27, 4, u8, u8, 8, {"gamma": True, "alpha": 0}),
    (0, 192, 108, 48, 27, 3, u16, f32, 16, {"gamma": True}),
    (1, 192, 108, 48, 27, 3, f32, u16, 16, {"gamma": True}),
    (2, 192, 108, 48, 27, 2, u16, u16, 16, {"gamma": True}),
    # bit-depth truncation, identity size, offsets, explicit k, negative k, other presets
    (0, 100, 60, 130, 97, 4, u8, u8, 6, {}),
    (1, 57, 33, 57, 33, 4, u8, u8, 8, {}),
    (1, 90, 70, 45, 35, 4, u8, u8, 8, {"ox": 0.37, "oy": -0.21}),
    (1, 90, 70, 45, 35, 4, u8, u8, 8, {"k": 2.0}),
    (2, 90, 70, 60, 45, 4, f32, f32, 16, {"k": -1.5}),
    (1, 96, 64, 48, 32, 4, u8, u8, 8, {"params": 1}),
    (2, 96, 64, 48, 32, 4, u8, u8, 8, {"params": 5}),
    # double image buffers: (float) cast in, (double) cast out (avir.h:2803-2806, 3168-3171);
    # double output of the default class takes the ordinary output stage, gamma included
    (1, 192, 108, 96, 54, 4, f64, f64, 16, {}),
    (2, 192, 108, 96, 54, 4, f64, f32, 16, {"buildmode": 1}),
    (0, 120, 80, 60, 40, 3, u8, f64, 8, {"gamma": True}),
    (0, 120, 80, 60, 40, 3, f32, f64, 16, {"gamma": True}),
    (1, 100, 60, 150, 77, 4, f64, u16, 16, {"gamma": True, "alpha": 3}),
    (2, 150, 90, 100, 55, 2, f64, u8, 8, {}),
    # error-diffusion ditherer (upstream CImageResizerDithererErrdINL / ErrdDIL composed into the
    # three classes: fpclass codes 3..5), integer output only; row-recursive
    (3, 120, 80, 60, 40, 4, u8, u8, 8, {}),
    (4, 120, 80, 60, 40, 4, u8, u8, 8, {}),
    (5, 120, 80, 60, 40, 4, u8, u8, 8, {}),
    (3, 100, 60, 150, 77, 3, u8, u8, 6, {}),                 # bit-depth truncation: TrMul != 1
    (4, 100, 60, 150, 97, 1, u16, u16, 12, {}),              # 3 row groups, one channel
    (5, 192, 108, 48, 27, 4, u8, u8, 5, {"gamma": True, "alpha": 3}),
    (3, 64, 48, 33, 70, 2, f32, u16, 16, {"gamma": True}),
    (4, 40, 30, 1, 65, 4, u8, u8, 8, {}),                    # one-pixel rows
    (5, 40, 30, 77, 1, 4, u8, u8, 8, {}),                    # one row
    (3, 120, 80, 60, 40, 4, u8, f32, 8, {}),                 # float output: the ditherer is skipped
    # tiny / ragged
    (1, 1, 1, 5, 7, 4, u8, u8, 8, {}),
    (1, 7, 5, 1, 1, 4, u8, u8, 8, {}),
    (2, 3, 200, 9, 50, 4, u8, u8, 8, {}),
    (0, 2, 2, 3, 3, 1, f32, f32, 16, {}),
]


def make_input(case, seed=7, structured=None):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    if structured is None:
        return o.lcg_image(sh, sw, ch, ti, seed=seed)
    mx = {u8: 255, u16: 65535, f32: 1.0, f64: 1.0}[ti]
    img = np.zeros((sh, sw, ch), dtype=ti)
    if structured == "ramp":
        xs = (np.arange(sw) / max(sw - 1, 1))[None, :, None]
        ys = (np.arange(sh) / max(sh - 1, 1))[:, None, None]
        img[:] = ((xs * 0.6 + ys * 0.4) * mx).astype(ti)
    elif structured == "impulse":
        for (y, x) in ((0, 0), (0, sw - 1), (sh - 1, 0), (sh - 1, sw - 1), (sh // 2, sw // 2)):
            img[y, x] = mx
    elif structured == "checker":
        yy, xx = np.mgrid[0:sh, 0:sw]
        img[((yy + xx) & 1) == 1] = mx
    return img


# ---- the value domain: samples outside [0, 1], non-finite, subnormal, on rounding ties ---------------

PATCH = 48  # constant patches: big enough that the filter output inside equals the patch value
F32_MAX = float(np.finfo(np.float32).max)
# patch values of the "huge" kind: far outside the output range, and either side of 2^31 once
# multiplied by OutMul = 255 (u8 output) and 65535 (u16 output) -- where (int) leaves int32
HUGE_VALUES = [1e6, -1e6, 1e8, -1e8, 1e30, -1e30]
for _m in (255.0, 65535.0):
    _b = np.float32(2.0 ** 31 / _m)
    for _v in (np.nextafter(_b, np.float32(0)), np.nextafter(_b, np.float32(np.inf))):
        HUGE_VALUES += [float(_v), -float(_v)]
NONFINITE_VALUES = [np.inf, -np.inf, -np.nan, 3e38, F32_MAX, -F32_MAX]
VALUE_KINDS = ("range", "huge", "nonfinite", "tiny", "ties")   # float sources
INT_KINDS = ("every_code", "zero", "max")                       # integer sources


def _patches(img, values, rng, size=PATCH):
    """size x size patches on a grid, at least `size` apart (a filter's reach at k <= 4: 1e30 in one
    patch must not swamp its neighbour), each channel of a patch constant at the next of `values`;
    (y, x, channel, value) of every patch centre."""
    sh, sw, ch = img.shape
    size = min(size, sh, sw)
    ny, nx = max(sh // (2 * size), 1), max(sw // (2 * size), 1)
    gy, gx = (sh - ny * size) // (ny + 1), (sw - nx * size) // (nx + 1)
    off = int(rng.integers(0, len(values)))
    centres = []
    for i in range(ny * nx):
        y0, x0 = gy + (i // nx) * (size + gy), gx + (i % nx) * (size + gx)
        for c in range(ch):
            v = values[(off + i * ch + c) % len(values)]
            img[y0:y0 + size, x0:x0 + size, c] = v
            centres.append((y0 + size // 2, x0 + size // 2, c, v))
    return centres


def _sparse(img, values, rng, count):
    """`count` single samples of `values` in turn at random positions and channels."""
    sh, sw, ch = img.shape
    for i in range(count):
        img[int(rng.integers(0, sh)), int(rng.integers(0, sw)), int(rng.integers(0, ch))] = values[i % len(values)]


def value_image(case, kind, seed=11):
    """A seeded source image of `kind` for the case's geometry and input type.

    Float sources (float32, or float64 with values beyond float32's range where noted):
      range      uniform in [-4, 4]: both sides of the output clamp, the sRGB polynomial outside [0, 1]
      huge       PATCH x PATCH constant patches of HUGE_VALUES on a [0, 1) background
      nonfinite  sparse +-Inf, a negative quiet NaN, 3e38 (where lin2srgb_batch_ok stops) and
                 +-FLT_MAX on a [0, 1) background
      tiny       subnormals of both signs down to 2^-149, +-0.0 and a few +-FLT_MIN
      ties       constant patches at (2k + 1) / (2 OutMul) and their float neighbours: outputs on
                 k + 0.5, where the rounding modes differ
    float64 sources add 1e39 / 1e300 (Inf once cast to float) and double subnormals.
    Integer sources:
      every_code every code of the type in every channel (u8: each channel 64 times over)
      zero, max  all-zero and all-maximum images."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    ti = np.dtype(ti)
    rng = np.random.default_rng(seed)
    if ti.kind != "f":
        mx = np.iinfo(ti).max
        if kind == "zero":
            return np.zeros((sh, sw, ch), ti)
        if kind == "max":
            return np.full((sh, sw, ch), mx, ti)
        assert kind == "every_code"
        n = sh * sw
        assert n >= mx + 1, "image too small for every code"
        img = np.empty((sh, sw, ch), ti)
        for c in range(ch):
            img[..., c] = rng.permutation(np.arange(n) % (mx + 1)).astype(ti).reshape(sh, sw)
        return img
    img = rng.random((sh, sw, ch))
    if kind == "range":
        img = rng.uniform(-4.0, 4.0, (sh, sw, ch))
    elif kind == "huge":
        _patches(img, HUGE_VALUES, rng)
    elif kind == "nonfinite":
        _sparse(img, NONFINITE_VALUES, rng, max(6, sh * sw // 1500))
    elif kind == "tiny":
        sub = rng.integers(0, 1 << 23, (sh, sw, ch)).astype(np.float64) * 2.0 ** -149
        sub[rng.random((sh, sw, ch)) < 0.1] = 0.0
        sub[rng.random((sh, sw, ch)) < 0.02] = 2.0 ** -126
        sub.ravel()[:8] = 2.0 ** -149
        img = np.where(rng.random((sh, sw, ch)) < 0.5, -sub, sub)
    elif kind == "ties":
        mul = {np.dtype(u8): 255.0, np.dtype(u16): 65535.0}.get(np.dtype(to), 255.0)
        levels = []
        for k_ in rng.integers(0, int(mul), 6):
            t = np.float32((2 * int(k_) + 1) / (2 * mul))
            levels += [float(np.nextafter(t, np.float32(-1))), float(t), float(np.nextafter(t, np.float32(2)))]
        _patches(img, levels, rng)
    else:
        raise ValueError(kind)
    if ti == np.float64:
        _sparse(img, [1e39, -1e39, 1e300, -1e300, 5e-324, -5e-324, 1e-310], rng, max(7, sh * sw // 1500))
        return img
    return img.astype(np.float32)


def huge_patch_centres(case, seed=11):
    """(y, x, channel, value) of the centres of value_image(case, "huge", seed)'s patches."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rng = np.random.default_rng(seed)
    img = rng.random((sh, sw, ch))
    return _patches(img, HUGE_VALUES, rng)


def value_mismatch(want, got):
    """Elements that differ: integers exactly; floats bit for bit except that any NaN matches any
    NaN (payloads are not preserved, positions are), so +-0 and +-Inf count."""
    assert want.shape == got.shape and want.dtype == got.dtype
    if want.dtype.kind != "f":
        return int((want != got).sum())
    nw_, ng = np.isnan(want), np.isnan(got)
    bits = np.uint32 if want.dtype == np.float32 else np.uint64
    differ = (want.view(bits) != got.view(bits)) & ~(nw_ & ng)
    return int(differ.sum())


def ref_kwargs(kw):
    return dict(k=kw.get("k", 0.0), ox=kw.get("ox", 0.0), oy=kw.get("oy", 0.0),
                gamma=kw.get("gamma", False), alpha=kw.get("alpha", -1),
                buildmode=kw.get("buildmode", -1), params=kw.get("params", 0))


def ref_output(case, src):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    return o.ref_resize(src, nw, nh, to, fpclass=fp, resbits=rb, **ref_kwargs(kw))


def resizer_and_vars(case):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs = ab.CImageResizer(rb, 0, kw.get("params", 0), fp)
    v = ab.CImageResizerVars(ox=kw.get("ox", 0.0), oy=kw.get("oy", 0.0),
                             UseSRGBGamma=kw.get("gamma", False), AlphaIndex=kw.get("alpha", -1),
                             BuildMode=kw.get("buildmode", -1))
    return rs, v


_port = None


def port():
    global _port
    if _port is None:
        lib = C.CDLL(os.path.join(ROOT, "oracle", "libavir_port.so"))
        for f in (lib.avir_port_resize, lib.lancir_port_resize):
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
            f.restype = C.c_int
        lib.avir_port_srgb_lut.argtypes = [C.c_void_p]
        _port = lib
    return _port


def port_output(case, src):
    """The C port executing the descriptor the product front-end builds."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = resizer_and_vars(case)
    h, dp, modes = rs.descriptor(src.shape, src.dtype, nw, nh, to, kw.get("k", 0.0), v)
    try:
        dst = np.zeros((nh, nw, ch), to)
        assert port().avir_port_resize(dp, src.ctypes.data, sw * ch, dst.ctypes.data, nw * ch) == 0
    finally:
        rs.free_descriptor(h)
    return dst, modes


def gpu_output(case, src):
    """The product: avir::CImageResizer<>::resizeImage through libavirb200.so."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = resizer_and_vars(case)
    return rs.resizeImage(src, nw, nh, kw.get("k", 0.0), v, out_dtype=to)


def count_mismatch(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype
    if a.dtype == np.float32:
        return int((a.view(np.uint32) != b.view(np.uint32)).sum())
    return int((a != b).sum())


# ---- caller layouts: padded pitches, offset bases, poisoned padding, guarded destinations ------------

SENTINEL = 0xA5  # every guard byte of a destination buffer
GUARD_ROWS = 2   # guard rows above and below a destination image


def poison_of(dtype):
    """Fill of a source buffer outside the image: a value no kernel may let into a result."""
    dtype = np.dtype(dtype)
    return np.nan if dtype.kind == "f" else np.iinfo(dtype).max


def image_view(backing, origin, pitch, shape):
    """(H, W, C) view of `backing` (1-D) starting at element `origin`, rows `pitch` elements apart."""
    h, w, c = shape
    it = backing.dtype.itemsize
    return np.lib.stride_tricks.as_strided(backing[origin:], shape=(h, w, c), strides=(pitch * it, c * it, it))


def host_array(n, dtype, pinned=False):
    """n elements of pageable (numpy) or page-locked (torch pin_memory) host memory."""
    dtype = np.dtype(dtype)
    if not pinned:
        return np.empty(n, dtype)
    import torch
    return torch.empty(n * dtype.itemsize, dtype=torch.uint8).pin_memory().numpy().view(dtype)


class Layout:
    """An image inside a larger 1-D buffer: `origin` (elements) of pixel (0, 0), `pitch` (elements)
    from one row to the next.  view() is the (H, W, C) image, is_outside() marks every byte of
    the buffer that is not part of it."""

    def __init__(self, backing, origin, pitch, shape):
        self.backing, self.origin, self.pitch, self.shape = backing, origin, pitch, tuple(shape)

    def view(self, backing=None):
        return image_view(self.backing if backing is None else backing, self.origin, self.pitch, self.shape)

    def outside_bytes(self, backing=None):
        """The bytes of (a copy of) the buffer outside the image, as a flat uint8 array."""
        b = (self.backing if backing is None else backing).view(np.uint8)
        inside = np.zeros(b.size, bool)
        h, w, c = self.shape
        it = self.backing.dtype.itemsize
        image_view(inside, self.origin * it, self.pitch * it, (h, w * c * it, 1))[:] = True
        return b[~inside]


def source_layout(img, extra_pitch=0, elem_offset=0, pinned=False):
    """`img` copied into a buffer with rows sw*C + extra_pitch elements apart, starting elem_offset
    elements in; every element outside the image holds poison_of(dtype)."""
    h, w, c = img.shape
    pitch = w * c + extra_pitch
    back = host_array(elem_offset + h * pitch + extra_pitch + 8, img.dtype, pinned)
    back[:] = poison_of(img.dtype)
    lay = Layout(back, elem_offset, pitch, img.shape)
    lay.view()[:] = img
    return lay


def guarded_dest(shape, dtype, extra_pitch=0, elem_offset=0, pinned=False):
    """A destination buffer for an (H, W, C) image: GUARD_ROWS rows above and below, rows
    W*C + extra_pitch elements apart, the image elem_offset elements into its row; every byte
    set to SENTINEL."""
    h, w, c = shape
    pitch = w * c + extra_pitch
    back = host_array((h + 2 * GUARD_ROWS) * pitch + elem_offset + 8, dtype, pinned)
    back.view(np.uint8)[:] = SENTINEL
    return Layout(back, GUARD_ROWS * pitch + elem_offset, pitch, shape)


def guard_damage(lay, backing=None):
    """Number of bytes outside the image that no longer hold SENTINEL."""
    return int((lay.outside_bytes(backing) != SENTINEL).sum())


def case_id(case):
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    s = "%s-%dx%d-%dx%d-c%d-%s-%s-b%d" % (("def", "f4", "dil", "defE", "f4E", "dilE")[fp], sw, sh, nw, nh, ch,
                                          np.dtype(ti).name, np.dtype(to).name, rb)
    for k_, v_ in sorted(kw.items()):
        s += "-%s%s" % (k_, v_)
    return s
