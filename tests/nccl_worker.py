"""Worker of tests/test_gpu_nccl.py (one process per GPU under torch.distributed.run): the real
NCCL-sharded path, avirb200_resize_sharded, against the 1-GPU avirb200_resize_device output of
the same image -- band by band, bit for bit (SURVEY.md section 4 tier 5; upstream avir.h:5797-5806
is why the plan must be the global one).  Exit code 0 = every case identical."""
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

u8, u16, f32 = np.uint8, np.uint16, np.float32
TT = {u8: torch.uint8, u16: torch.uint16, f32: torch.float32}

CASES = [
    (2, 1920, 2160, 960, 1080, 4, f32, f32, 16, {}),                 # cfg3 chain (streaming kernel)
    (1, 4096, 4096, 1024, 1024, 4, u16, u16, 16, {}),                # cfg4 chain
    (2, 1920, 2160, 480, 540, 4, u8, u8, 8, {"gamma": True, "alpha": 3}),  # cfg5 chain (tile kernel)
    (1, 960, 1080, 1920, 2160, 4, u8, u8, 8, {}),                    # cfg2: upsizing
    (0, 700, 900, 431, 557, 3, u8, u8, 8, {}),                       # generic kernel, odd ratio, RGB
    # RGB widened onto the 4-channel kernels, both passes forced onto the generic kernel: the halo rows
    # and band offsets of a 4-float intermediate
    (0, 1280, 1440, 640, 720, 3, u8, u8, 8, {"family": 1}),
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
    lib.avirb200_resize_sharded.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                            C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    lib.avirb200_resize_device.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t,
                                           C.c_void_p, C.c_void_p]
    lib.avirb200_plan_set_option.argtypes = [C.c_void_p, C.c_int, C.c_int]
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
    overlaps = [int(v) for v in os.environ.get("AVIR_NCCL_OVERLAPS", "3,1,2,0").split(",")]
    debug = os.environ.get("AVIR_NCCL_DEBUG") == "1"

    def dbg(*a):
        if debug:
            torch.cuda.synchronize()
            print("[rank %d]" % rank, *a, flush=True)
    ncases = int(os.environ.get("AVIR_NCCL_CASES", "0")) or len(CASES)
    for case in CASES[:ncases]:
        for overlap in overlaps:
            fp, sw, sh, nw, nh, ch, ti, to, rb, kw = case
            src = cs.make_input(case, seed=77)  # same image on every rank
            rs, v = cs.resizer_and_vars(case)
            h, dp, _ = rs.descriptor(src.shape, ti, nw, nh, to, 0.0, v)
            plan = C.c_void_p()
            assert lib.avirb200_plan_create(C.c_void_p(dp), C.byref(plan)) == 0, lib.avirb200_last_error()
            assert lib.avirb200_plan_set_option(plan, ab.OPT_OVERLAP_HALO, overlap) == 0
            assert lib.avirb200_plan_set_option(plan, ab.OPT_KERNEL_FAMILY, kw.get("family", 0)) == 0
            si = SI()
            assert lib.avirb200_shard_query(plan, rank, world, C.byref(si)) == 0, lib.avirb200_last_error()
            wsb, wsf = C.c_size_t(), C.c_size_t()
            assert lib.avirb200_shard_workspace_bytes(plan, rank, world, C.byref(wsb)) == 0
            assert lib.avirb200_plan_workspace_bytes(plan, C.byref(wsf)) == 0
            d_all = torch.from_numpy(src).cuda()
            d_band = d_all[si.src_row0:si.src_row0 + si.src_rows].contiguous()
            d_dst = torch.zeros((si.dst_rows, nw, ch), device="cuda", dtype=TT[to])
            d_ws = torch.empty(wsb.value, dtype=torch.uint8, device="cuda")
            dbg("plan ready", cs.case_id(case), "overlap", overlap, "halo", si.halo_up, si.halo_down, "ws", wsb.value)
            for it in range(2):  # twice: the second call reuses the exchange buffers / flags
                assert lib.avirb200_resize_sharded(plan, comm, rank, world, d_band.data_ptr(), sw * ch,
                                                   d_dst.data_ptr(), nw * ch, d_ws.data_ptr(), st) == 0, \
                    lib.avirb200_last_error()
                dbg("sharded call", it, "done")
            torch.cuda.synchronize()
            whole = torch.zeros((nh, nw, ch), device="cuda", dtype=TT[to])
            ws2 = torch.empty(wsf.value, dtype=torch.uint8, device="cuda")
            assert lib.avirb200_resize_device(plan, d_all.data_ptr(), sw * ch, whole.data_ptr(), nw * ch,
                                              ws2.data_ptr(), st) == 0
            torch.cuda.synchronize()
            mine = whole[si.dst_row0:si.dst_row0 + si.dst_rows]
            a = mine.contiguous().view(torch.uint8)
            b = d_dst.view(torch.uint8)
            n = torch.tensor([int((a != b).sum().item())], device="cuda")
            dist.all_reduce(n)
            if rank == 0:
                print("%s overlap=%d ranks=%d halo=%d/%d mismatches=%d" % (cs.case_id(case), overlap, world,
                                                                          si.halo_up, si.halo_down, int(n.item())), flush=True)
            bad += int(n.item())
            dist.barrier()  # (a rank's mailbox is freed only after every rank is done with the case)
            lib.avirb200_plan_destroy(plan)
            rs.free_descriptor(h)
            dbg("plan destroyed")
    lib.avirb200_comm_destroy(comm)
    dist.destroy_process_group()
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
