"""Worker of tests/test_gpu_lancir_sharded.py (one process per GPU under torch.distributed.run):
lancirb200_resize_sharded against the 1-GPU lancirb200_resize_device of the same image, band by band, bit for
bit, on the mailbox (3) and NCCL (0) schedules.  Two calls per plan with different sources use both mailbox
slots; the third reuses the first slot.  Exit code 0 = every case identical."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import avir_b200 as ab  # noqa: E402

u8, u16, f32, f64, u32 = np.uint8, np.uint16, np.float32, np.float64, np.uint32
CODE = {np.dtype(t): k for k, t in enumerate((u8, u16, f32, f64, u32))}  # avirb200_dtype

# (sw, sh, nw, nh, channels, Tin, Tout, CLancIRParams fields)
CASES = [
    (7680, 4320, 3840, 2160, 4, u8, u8, {}),               # the headline: k = 2, vector kernels
    (1920, 1080, 1281, 1711, 4, u16, f32, {}),              # upsizing vertically
    (999, 733, 517, 301, 3, f32, u8, {"oy": 3.5}),          # scalar kernels, offset
    (640, 960, 320, 480, 4, f64, u32, {"kx": 3.0}),
    (512, 2048, 500, 1000, 1, u32, f64, {"la": 5.0, "oy": -7.25}),
    (400, 800, 400, 800, 2, f32, u16, {"oy": -2.25}),    # rows travel one way only: NCCL on every pair
]


def descriptor(case):
    """(handle, descriptor pointer) of the case as CLancIR::resizeImage builds it; free with
    lancirb200_host_desc_free(handle)."""
    sw, sh, nw, nh, ch, ti, to, kw = case
    h = ab.host_lib().lancirb200_host_desc_create(CODE[np.dtype(ti)], CODE[np.dtype(to)], sw, sh, nw, nh, ch,
                                                  kw.get("kx", 0.0), kw.get("ky", 0.0), kw.get("ox", 0.0),
                                                  kw.get("oy", 0.0), kw.get("la", 3.0))
    assert h, ab.host_lib().avirb200_host_last_error()
    return h, ab.host_lib().lancirb200_host_desc_get(h)


class SI(C.Structure):
    _fields_ = [(n_, C.c_int32) for n_ in ("src_row0", "src_rows", "dst_row0", "dst_rows",
                                           "need_row0", "need_rows", "halo_up", "halo_down")]


def main():
    import torch
    import torch.distributed as dist
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib = ab.lib()
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    lib.lancirb200_resize_sharded.argtypes = [vp, vp, i, i, vp, sz, vp, sz, vp, vp]
    lib.lancirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    lib.lancirb200_plan_set_option.argtypes = [vp, i, i]
    lib.lancirb200_shard_query.argtypes = [vp, i, i, vp]
    lib.lancirb200_shard_workspace_bytes.argtypes = [vp, i, i, vp]
    lib.lancirb200_plan_workspace_bytes.argtypes = [vp, vp]
    idbuf = torch.zeros(128, dtype=torch.uint8)
    if rank == 0:
        raw = (C.c_char * 128)()
        assert lib.avirb200_comm_unique_id(raw) == 0, lib.avirb200_last_error()
        idbuf = torch.frombuffer(bytearray(raw.raw), dtype=torch.uint8).clone()
    idg = idbuf.cuda()
    dist.broadcast(idg, 0)
    raw = (C.c_char * 128).from_buffer_copy(bytes(idg.cpu().numpy().tobytes()))
    comm = C.c_void_p()
    assert lib.avirb200_comm_create(raw, rank, world, C.byref(comm)) == 0, lib.avirb200_last_error()
    st = torch.cuda.current_stream().cuda_stream
    bad = 0
    for case in CASES:
        sw, sh, nw, nh, ch, ti, to, kw = case
        for overlap in (3, 0):
            h, dp = descriptor(case)
            plan = C.c_void_p()
            assert lib.lancirb200_plan_create(C.c_void_p(dp), C.byref(plan)) == 0, lib.avirb200_last_error()
            assert lib.lancirb200_plan_set_option(plan, ab.OPT_OVERLAP_HALO, overlap) == 0
            si = SI()
            assert lib.lancirb200_shard_query(plan, rank, world, C.byref(si)) == 0, lib.avirb200_last_error()
            wsb, wsf = C.c_size_t(), C.c_size_t()
            assert lib.lancirb200_shard_workspace_bytes(plan, rank, world, C.byref(wsb)) == 0
            assert lib.lancirb200_plan_workspace_bytes(plan, C.byref(wsf)) == 0
            d_ws = torch.empty(wsb.value, dtype=torch.uint8, device="cuda")
            ws2 = torch.empty(wsf.value, dtype=torch.uint8, device="cuda")
            isz, osz = np.dtype(ti).itemsize, np.dtype(to).itemsize
            n = 0
            for call in range(3):  # consecutive calls, new sources: both mailbox slots, the first one reused
                g = torch.Generator(device="cuda").manual_seed(91 + call)   # same image on every rank
                d_all = torch.randint(0, 256, (sh * sw * ch * isz,), generator=g, device="cuda",
                                      dtype=torch.int32).to(torch.uint8)
                if ti in (f32, f64):   # finite values in [0, 1)
                    vals = torch.rand(sh * sw * ch, generator=g, device="cuda",
                                      dtype=torch.float32 if ti == f32 else torch.float64)
                    d_all = vals.view(torch.uint8).clone()
                band = d_all.view(sh, -1)[si.src_row0:si.src_row0 + si.src_rows].contiguous()
                d_dst = torch.zeros(si.dst_rows * nw * ch * osz, device="cuda", dtype=torch.uint8)
                assert lib.lancirb200_resize_sharded(plan, comm, rank, world, band.data_ptr(), sw * ch,
                                                     d_dst.data_ptr(), nw * ch, d_ws.data_ptr(), st) == 0, \
                    lib.avirb200_last_error()
                whole = torch.zeros(nh * nw * ch * osz, device="cuda", dtype=torch.uint8)
                assert lib.lancirb200_resize_device(plan, d_all.data_ptr(), sw * ch, whole.data_ptr(), nw * ch,
                                                    ws2.data_ptr(), st) == 0
                torch.cuda.synchronize()
                mine = whole.view(nh, -1)[si.dst_row0:si.dst_row0 + si.dst_rows].reshape(-1)
                n += int((mine != d_dst).sum().item())
            t = torch.tensor([n], device="cuda")
            dist.all_reduce(t)
            if rank == 0:
                print("%dx%d-%dx%d-c%d overlap=%d ranks=%d mismatches=%d" % (sw, sh, nw, nh, ch, overlap, world,
                                                                            int(t.item())), flush=True)
            bad += int(t.item())
            dist.barrier()  # (a rank's mailbox is freed only after every rank is done with the case)
            lib.lancirb200_plan_destroy(plan)
            ab.host_lib().lancirb200_host_desc_free(h)
    lib.avirb200_comm_destroy(comm)
    dist.destroy_process_group()
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
