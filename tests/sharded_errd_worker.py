"""Worker of tests/test_gpu_sharded_errd.py (one process per GPU under torch.distributed.run):
avirb200_resize_sharded with double buffers and error diffusion against the 1-GPU avirb200_resize_device of
the same image, band by band, bit for bit, on the fused (3), push (1) and NCCL (0) schedules.  Three calls
per plan with different sources exercise both mailbox slots.  Exit code 0 = every case identical."""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import avir_b200 as ab  # noqa: E402
import cases as cs  # noqa: E402

u8, u16, f32, f64 = np.uint8, np.uint16, np.float32, np.float64

CASES = [
    (5, 1920, 2160, 480, 540, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),  # cfg5 chain, dithered
    (4, 1024, 1024, 256, 256, 4, u16, u16, 16, {}),                      # cfg4 chain, dithered
    (3, 700, 900, 431, 557, 3, u8, u8, 8, {}),                           # default class, RGB, dithered
    (2, 1920, 2160, 960, 1080, 4, f64, f64, 16, {}),                     # cfg3 chain on double buffers
    (5, 1280, 1440, 640, 720, 4, f64, u8, 8, {}),                        # double source, dithered output
]


class SI(C.Structure):
    _fields_ = [(n_, C.c_int32) for n_ in ("src_row0", "src_rows", "dst_row0", "dst_rows",
                                           "need_row0", "need_rows", "halo_up", "halo_down")]


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib = ab.lib()
    vp, sz = C.c_void_p, C.c_size_t
    lib.avirb200_resize_sharded.argtypes = [vp, vp, C.c_int, C.c_int, vp, sz, vp, sz, vp, vp]
    lib.avirb200_resize_device.argtypes = [vp, vp, sz, vp, sz, vp, vp]
    lib.avirb200_plan_set_option.argtypes = [vp, C.c_int, C.c_int]
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
        for overlap in (3, 1, 0):
            fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
            rs, v = cs.resizer_and_vars(case)
            h, dp, _ = rs.descriptor((sh, sw, ch), ti, nw, nh, to, 0.0, v)
            plan = C.c_void_p()
            assert lib.avirb200_plan_create(C.c_void_p(dp), C.byref(plan)) == 0, lib.avirb200_last_error()
            assert lib.avirb200_plan_set_option(plan, ab.OPT_OVERLAP_HALO, overlap) == 0
            si = SI()
            assert lib.avirb200_shard_query(plan, rank, world, C.byref(si)) == 0, lib.avirb200_last_error()
            wsb, wsf = C.c_size_t(), C.c_size_t()
            assert lib.avirb200_shard_workspace_bytes(plan, rank, world, C.byref(wsb)) == 0
            assert lib.avirb200_plan_workspace_bytes(plan, C.byref(wsf)) == 0
            d_ws = torch.empty(wsb.value, dtype=torch.uint8, device="cuda")
            ws2 = torch.empty(wsf.value, dtype=torch.uint8, device="cuda")
            osz = np.dtype(to).itemsize
            n = 0
            for call in range(3):  # consecutive calls, new sources: both mailbox slots, the second one reused
                src = np.ascontiguousarray(cs.make_input(case, seed=77 + call))  # same image on every rank
                d_all = torch.from_numpy(src.view(np.uint8)).cuda()
                band = d_all.view(sh, -1)[si.src_row0:si.src_row0 + si.src_rows].contiguous()
                d_dst = torch.zeros(si.dst_rows * nw * ch * osz, device="cuda", dtype=torch.uint8)
                assert lib.avirb200_resize_sharded(plan, comm, rank, world, band.data_ptr(), sw * ch, d_dst.data_ptr(),
                                                   nw * ch, d_ws.data_ptr(), st) == 0, lib.avirb200_last_error()
                whole = torch.zeros(nh * nw * ch * osz, device="cuda", dtype=torch.uint8)
                assert lib.avirb200_resize_device(plan, d_all.data_ptr(), sw * ch, whole.data_ptr(), nw * ch,
                                                  ws2.data_ptr(), st) == 0
                torch.cuda.synchronize()
                mine = whole.view(nh, -1)[si.dst_row0:si.dst_row0 + si.dst_rows].reshape(-1)
                n += int((mine != d_dst).sum().item())
            t = torch.tensor([n], device="cuda")
            dist.all_reduce(t)
            if rank == 0:
                print("%s overlap=%d ranks=%d mismatches=%d" % (cs.case_id(case), overlap, world, int(t.item())),
                      flush=True)
            bad += int(t.item())
            dist.barrier()  # (a rank's mailbox is freed only after every rank is done with the case)
            lib.avirb200_plan_destroy(plan)
            rs.free_descriptor(h)
    lib.avirb200_comm_destroy(comm)
    dist.destroy_process_group()
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
