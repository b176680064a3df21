"""C2C plans with axis lengths that are not powers of two on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_nonpow2.py

For slab and pencil plans, Peer2Peer and All2All, Sync and Streams (which runs the sequential schedule for these lengths),
f64 and f32: every rank runs single-GPU cuFFT (oracle/_ref/libcufft_ref.so, built by `make -C oracle`) on the whole
seeded array and compares its own block of the forward output, then checks the inverse round trip of its block."""
import ctypes as C
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
SYNC, STREAMS = dfft.SendMethod.Sync, dfft.SendMethod.Streams


def cufft():
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libcufft_ref.so"))
    lib.cufft_ref_3d.restype = C.c_int
    lib.cufft_ref_3d.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int]
    return lib


def rel(a, b):
    return float((a - b).abs().pow(2).sum().sqrt() / b.abs().pow(2).sum().sqrt())


def blk(a, size, start):
    return a[start[0]:start[0] + size[0], start[1]:start[1] + size[1], start[2]:start[2] + size[2]]


def check(comm, world, rank, decomp, comm_method, send, f64, shape, ref_lib):
    cfg = dfft.Configurations(comm_method=comm_method, send_method=send, comm_method2=comm_method, send_method2=send)
    prec = "double" if f64 else "float"
    if decomp == "slab":
        p1, p2 = world, 1
        plan = dfft.MPIcuFFT_Slab(cfg, comm, precision=prec, transform="c2c")
        plan.initFFT(dfft.GlobalSize(*shape), None, True)
        dec = dfft.SLAB_ZY_THEN_X
    else:
        p1 = 2 if world % 2 == 0 else 1
        p2 = world // p1
        plan = dfft.MPIcuFFT_Pencil(cfg, comm, precision=prec, transform="c2c")
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, p2), True)
        dec = dfft.PENCIL
    rdt = torch.float64 if f64 else torch.float32
    cdt = torch.complex128 if f64 else torch.complex64
    g = torch.Generator(device="cuda").manual_seed(5)
    xg = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
    ref = torch.empty_like(xg)
    ms = C.c_float()
    assert ref_lib.cufft_ref_3d(1 if f64 else 0, 0, *shape, ref.data_ptr(), xg.data_ptr(), C.byref(ms), 1) == 0
    isz, ist = dfft.layout(dec, dfft.C2C, *shape, p1, p2, rank, 0)
    osz, ost = dfft.layout(dec, dfft.C2C, *shape, p1, p2, rank, 3)
    x = blk(xg, isz, ist).contiguous()
    spec = torch.empty(plan.getDomainSize() // (16 if f64 else 8), dtype=cdt, device="cuda")
    back = torch.empty_like(x)
    plan.execC2C(spec, x, dfft.FORWARD)
    n_out = osz[0] * osz[1] * osz[2]
    tol = 1e-10 if f64 else 1e-5
    ok = rel(spec[:n_out].reshape(osz), blk(ref, osz, ost)) < tol
    plan.execC2C(back, spec, dfft.INVERSE)
    ok &= rel(back / float(shape[0] * shape[1] * shape[2]), x) < tol
    plan.destroy()
    t = torch.tensor([0.0 if ok else 1.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item() == 0


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = dfft.Comm.from_torch_distributed(local)
    ref_lib = cufft()
    fails = 0
    for shape in ((100, 120, 90), (96, 64, 7 * world)):
        for decomp in ("slab", "pencil"):
            for comm_method in (P2P, A2A):
                for send in (SYNC, STREAMS):
                    for f64 in (True, False):
                        ok = check(comm, world, rank, decomp, comm_method, send, f64, shape, ref_lib)
                        if rank == 0:
                            print(f"{'ok  ' if ok else 'FAIL'} {shape} {decomp} {comm_method.name} {send.name} {'f64' if f64 else 'f32'}", flush=True)
                        fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_nonpow2: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
