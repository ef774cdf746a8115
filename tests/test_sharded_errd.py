"""Error diffusion across bands, on the CPU.

A sharded call dithers each band with errd_kernel: the band's first 32-row group starts from the D row the
band above left (instead of zeros), and the band's last row publishes the D row below it for the band below.
Here errd_kernel's systolic schedule is emulated in lockstep (lane = row of a 32-row group, lane l works on
pixel t - 2l at step t, D values move one lane down per step; a group's lane 0 takes them from the group
above, or from the carried row), band by band, and the bands' outputs must equal the C port's whole-image
ditherer element for element.  The band edges fall inside and on group edges, one band is a single row, and
the de-interleaved class's last-pixel quirk (pixel 0 of plane c+1 feeds plane c's last D) crosses every edge.

The workspace and mailbox arithmetic of double and error-diffusion plans is restated in Python as well
(shard_workspace_bytes, mailbox_bytes) and compared with the library's (avirb200_shard_layout_desc, host
arithmetic); the GPU tests compare that with avirb200_shard_workspace_bytes of created plans."""
import ctypes as C

import numpy as np
import pytest

import avir_b200 as ab
import cases as cs

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64
F = np.float32
C1, C2, C3 = F(0.364842), F(0.207305), F(0.063011)
OUT_TYPE_OFFSET = 24  # avirb200_plan_desc.out_type (after src_w, src_h, dst_w, dst_h, channels, in_type)
F32_CODE = 2


class DescHead(C.Structure):
    """The scalar head of avirb200_plan_desc (include/avirb200.h)."""
    _fields_ = [(n, C.c_int32) for n in ("src_w", "src_h", "dst_w", "dst_h", "channels", "in_type", "out_type",
                                          "sum_mode", "round_mode", "use_gamma", "alpha_index")] + \
               [(n, C.c_float) for n in ("in_gamma_mult", "out_gamma_mult", "tr_mul", "tr_mul_inv", "pk_out")] + \
               [("dither", C.c_int32)]


def _round(v, mode):
    """round_out / the port's round_mode for one float32."""
    v = F(v)
    if mode == 0:
        return -F(int(F(F(0.5) - v))) if v < 0 else F(int(F(v + F(0.5))))
    if mode == 1:
        if not (-2147483648.0 <= v < 2147483648.0):
            return F(-2147483648.0)
        return F(np.rint(v))
    return F(np.rint(v))


def errd_band(v, head, carry_in=None):
    """errd_kernel over one band's float rows v [H][W][C] in lockstep: (output, D row below the last row).
    carry_in: the D row of the band above (None: zeros, the image's first row)."""
    H, W, Ch = v.shape
    out = np.zeros((H, W, Ch), np.float32)
    planar = head.sum_mode == 1
    tr_mul, tr_inv, pk = F(head.tr_mul), F(head.tr_mul_inv), F(head.pk_out)
    above = None  # the D row the previous group's last row published
    for g in range((H + 31) // 32):
        lanes = min(32, H - g * 32)
        nm1, c3p, part, dn, n2first = (np.zeros((32, Ch), F) for _ in range(5))
        pub = np.zeros((W, Ch), F)
        for t in range(W + 2 * 31 + 1):
            din_all = np.zeros((32, Ch), F)
            din_all[1:] = dn[:-1]  # __shfl_up_sync of the previous step's dn
            for lane in range(lanes):
                pix = t - 2 * lane
                y = g * 32 + lane
                if 0 <= pix < W:
                    if lane > 0:
                        din = din_all[lane]
                    elif g > 0:
                        din = above[pix]
                    elif carry_in is not None:
                        din = carry_in[pix]
                    else:
                        din = np.zeros(Ch, F)
                    for c in range(Ch):
                        R = F(v[y, pix, c] + din[c])
                        if pix > 0:
                            R = F(R + nm1[lane, c])
                        z0 = F(_round(F(R * tr_inv), head.round_mode) * tr_mul)
                        noise = F(R - z0)
                        out[y, pix, c] = F(0) if z0 < 0 else (pk if z0 > pk else z0)
                        n1, n2, n3 = F(noise * C1), F(noise * C2), F(noise * C3)
                        if pix == 0:
                            n2first[lane, c] = n2
                        dn[lane, c] = F(part[lane, c] + n2)
                        part[lane, c] = F(F(0) + n1) if pix == 0 else F(F(F(0) + c3p[lane, c]) + n1)
                        c3p[lane, c] = n3
                        nm1[lane, c] = n1
                    q = pix - 1
                elif pix == W:
                    for c in range(Ch):
                        dn[lane, c] = part[lane, c]
                        if planar and c + 1 < Ch:
                            dn[lane, c] = F(dn[lane, c] + n2first[lane, c + 1])
                    q = W - 1
                else:
                    q = -1
                if lane == lanes - 1 and q >= 0:  # the group's last row: lane 31, or the band's last row
                    pub[q] = dn[lane]
        above = pub
    return out, above


def dither_floats(case, seed=3):
    """(the float rows the ditherer starts from, the C port's whole-image dithered output, descriptor head)."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    src = cs.make_input(case, seed=seed)
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor(src.shape, ti, nw, nh, to, kw.get("k", 0.0), v)
    try:
        head = DescHead.from_address(dp)
        assert head.dither == 1 and head.out_type in (0, 1), "not an error-diffusion plan"
        want = np.zeros((nh, nw, ch), to)
        assert cs.port().avir_port_resize(dp, src.ctypes.data, sw * ch, want.ctypes.data, nw * ch) == 0
        # the same descriptor with float output: the port's gamma-corrected rows, before any rounding
        io_out = head.out_type
        head.out_type = F32_CODE
        rows = np.zeros((nh, nw, ch), np.float32)
        try:
            assert cs.port().avir_port_resize(dp, src.ctypes.data, sw * ch, rows.ctypes.data, nw * ch) == 0
        finally:
            head.out_type = io_out
        frozen = DescHead.from_buffer_copy(head)
    finally:
        rs.free_descriptor(h)
    return rows, want, frozen


def banded(rows, head, edges):
    """errd_band over the bands [edges[i], edges[i+1]), each starting from the D row the band above left."""
    outs, carry = [], None
    for a, b in zip(edges, edges[1:]):
        o, carry = errd_band(rows[a:b], head, carry)
        outs.append(o)
    return np.concatenate(outs)


# destination heights and band edges: edges on and inside 32-row group edges, a one-row band
BANDS = {
    2: [0, 32, 70],
    3: [0, 20, 21, 70],
    5: [0, 13, 31, 33, 64, 70],
}
# (fpclass 3 / 4 / 5: the error-diffusion forms of the three classes) x channels x output types
ERRD_CASES = [(fp, 96, 140, 23, 70, ch, u8, u8, 8, {}) for fp in (3, 4, 5) for ch in (1, 2, 3, 4)] + [
    (5, 96, 140, 23, 70, 4, u16, u16, 16, {}),                              # u16 output
    (4, 96, 140, 23, 70, 3, u8, u8, 6, {}),                                 # bit-depth truncation
    (5, 96, 140, 23, 70, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),        # sRGB gamma, alpha last
    (3, 96, 140, 23, 70, 4, u8, u8, 8, {"gamma": True, "alpha": 0}),        # alpha first
]


@pytest.mark.parametrize("nbands", sorted(BANDS))
@pytest.mark.parametrize("case", ERRD_CASES, ids=cs.case_id)
def test_banded_ditherer_matches_whole_image_port(case, nbands):
    rows, want, head = dither_floats(case)
    got = banded(rows, head, BANDS[nbands]).astype(want.dtype)
    assert cs.count_mismatch(want, got) == 0


def test_lockstep_emulation_is_the_port_on_one_band():
    """The emulation itself, unbanded, is the port (so a banded mismatch is the handoff's)."""
    rows, want, head = dither_floats(ERRD_CASES[11])
    assert cs.count_mismatch(want, errd_band(rows, head)[0].astype(want.dtype)) == 0


def test_carry_is_what_the_next_band_needs():
    """The carried row is the D row of the band's next row: zeros instead of it change the next band."""
    rows, want, head = dither_floats(ERRD_CASES[11])
    top, carry = errd_band(rows[:32], head)
    assert np.any(carry != 0)
    lost = errd_band(rows[32:], head)[0].astype(want.dtype)
    assert cs.count_mismatch(want[32:], lost) > 0


# ---- workspace and mailbox arithmetic ---------------------------------------------------------------------

def _a256(n):
    return (n + 255) // 256 * 256


def shard_workspace_bytes(si, src_w, dst_w, ch, f64_in, f64_out, errd):
    """avirb200_shard_workspace_bytes of a plan with double buffers or error diffusion (never widened to 4
    channels): the intermediate, the band's float source copy (in32), its float destination rows (out32), the
    ditherer's boundary rows and counters per 32-row group of the band, and the two carried D rows."""
    n = _a256(si["need_rows"] * dst_w * ch * 4)
    if f64_in:
        n += _a256(src_w * si["src_rows"] * ch * 4)
    if f64_out or errd:
        n += _a256(dst_w * si["dst_rows"] * ch * 4)
    if errd:
        groups = (si["dst_rows"] + 31) // 32
        n += _a256(groups * dst_w * ch * 4) + _a256(groups * 4) + _a256(2 * dst_w * ch * 4)
    return n


def mailbox_bytes(si, dst_w, ch, errd, slots):
    """MailboxLayout::bytes: the 256-byte header, then per slot the halo rows from above and below and, for
    error diffusion, the D row from the band above."""
    slot = _a256(si["halo_up"] * dst_w * ch * 4) + _a256(si["halo_down"] * dst_w * ch * 4)
    if errd:
        slot += _a256(dst_w * ch * 4)
    return 256 + slots * slot


def shard_layout(case, rank, nranks):
    """(code, workspace bytes, mailbox bytes, shard info dict) from avirb200_shard_layout_desc and
    avirb200_shard_query_desc: the library's ws_layout and MailboxLayout, no device needed."""
    from test_sharding import shard_info
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    rs, v = cs.resizer_and_vars(case)
    h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, kw.get("k", 0.0), v)
    try:
        L = ab.lib()
        L.avirb200_shard_layout_desc.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        ws, box = C.c_size_t(), C.c_size_t()
        r = L.avirb200_shard_layout_desc(C.c_void_p(dp), rank, nranks, C.byref(ws), C.byref(box))
        _, si = shard_info(dp, rank, nranks)
    finally:
        rs.free_descriptor(h)
    return r, ws.value, box.value, {k: getattr(si, k) for k, _ in si._fields_}


LAYOUT_CASES = [
    (5, 640, 720, 320, 360, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),   # error diffusion
    (4, 640, 720, 320, 360, 3, u16, u16, 16, {}),                         # error diffusion, RGB
    (3, 640, 720, 320, 360, 1, u8, u8, 6, {}),                            # error diffusion, gray, truncation
    (1, 640, 720, 320, 360, 4, f64, f64, 16, {}),                         # double in and out
    (2, 640, 720, 320, 360, 3, f64, u8, 8, {}),                           # double in
    (1, 640, 720, 320, 360, 2, u8, f64, 8, {}),                           # double out
    (5, 640, 720, 320, 360, 4, f64, u16, 16, {}),                         # double in, dithered out
    (2, 640, 720, 320, 360, 4, f32, f32, 16, {}),                         # neither: 4 channels
]


@pytest.mark.parametrize("nranks", [2, 5, 8])
@pytest.mark.parametrize("case", LAYOUT_CASES, ids=cs.case_id)
def test_shard_workspace_and_mailbox_sizes_match_the_library(case, nranks):
    """Every rank's workspace and mailbox bytes as ws_layout and MailboxLayout compute them (through
    avirb200_shard_layout_desc) equal the arithmetic restated above."""
    fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
    errd = fp >= 3 and np.dtype(to).kind != "f"
    for rank in range(nranks):
        r, ws, box, si = shard_layout(case, rank, nranks)
        assert r == 0, (rank, ab.lib().avirb200_last_error())
        assert ws == shard_workspace_bytes(si, sw, nw, ch, np.dtype(ti) == f64, np.dtype(to) == f64, errd), rank
        assert box == mailbox_bytes(si, nw, ch, errd, 2), rank


def test_shard_layout_refuses_plans_that_may_be_widened():
    """A 1..3-channel plan without double buffers or error diffusion may run on the 4-channel kernels, which
    plan creation decides: the descriptor alone does not give its layout."""
    assert shard_layout((0, 320, 360, 160, 180, 3, u8, u8, 8, {}), 0, 2)[0] == -4


def test_workspace_arithmetic_follows_the_band():
    """A band's double and error-diffusion segments are the band's, not the image's: 8 bands of a 1080-row
    destination need about an eighth of the whole image's out32 each."""
    whole = dict(need_rows=4320, src_rows=4320, dst_rows=1080)
    band = dict(need_rows=560, src_rows=540, dst_rows=135)
    a = shard_workspace_bytes(whole, 7680, 1920, 4, True, False, True)
    b = shard_workspace_bytes(band, 7680, 1920, 4, True, False, True)
    assert 7 * b < a < 9 * b
