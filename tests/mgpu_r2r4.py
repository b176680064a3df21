"""Plans with type-IV kinds (DCT-IV / DST-IV) on several GPUs (run under torchrun with 2-8 GPUs):

    torchrun --nproc-per-node N tests/mgpu_r2r4.py

For slab, Z_Then_YX and pencil plans, Peer2Peer and All2All, Sync and Streams (which runs the sequential schedule for these
plans), type-IV / type-I / type-II / R2HC mixes and f64 / f32: every rank regenerates the seeded global array, compares its
own block of the forward output with the per-axis transform of the whole array (scipy's dct / dst, type=4 on type-IV
axes), then checks the inverse through the round trip of its block, which scales by 2N per type-IV, type-I, DCT and DST
axis (N = L - 1 for DCT-I, L + 1 for DST-I) and N per R2HC axis."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import distributedfft_b200 as dfft  # noqa: E402
from test_r2r4 import global_ref, shape_for  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
SYNC, STREAMS = dfft.SendMethod.Sync, dfft.SendMethod.Streams
KIND = {"dct": dfft.DCT, "dst": dfft.DST, "r2hc": dfft.R2HC, "dct1": dfft.DCT1, "dst1": dfft.DST1, "dct4": dfft.DCT4, "dst4": dfft.DST4}
PER_AXIS = {"r2hc": 1, "dct": 2, "dst": 2, "dct1": 2, "dst1": 2, "dct4": 2, "dst4": 2}
N_OF = {"dct1": -1, "dst1": 1}  # N = L + N_OF on type-I axes


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def blk(a, size, start):
    return a[start[0]:start[0] + size[0], start[1]:start[1] + size[1], start[2]:start[2] + size[2]]


def check(comm, world, rank, decomp, names, comm_method, send, f64, base):
    shape = shape_for(base, tuple(KIND[k] for k in names))
    cfg = dfft.Configurations(comm_method=comm_method, send_method=send, comm_method2=comm_method, send_method2=send)
    prec = "double" if f64 else "float"
    if decomp == "pencil":
        p1 = 2 if world % 2 == 0 else 1
        p2 = world // p1
        plan = dfft.MPIcuFFT_Pencil(cfg, comm, precision=prec, transform=names)
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, p2), True)
        dec = dfft.PENCIL
    else:
        p1, p2 = world, 1
        cls = dfft.MPIcuFFT_Slab if decomp == "slab" else dfft.MPIcuFFT_Slab_Z_Then_YX
        plan = cls(cfg, comm, precision=prec, transform=names)
        plan.initFFT(dfft.GlobalSize(*shape), None, True)
        dec = dfft.SLAB_ZY_THEN_X if decomp == "slab" else dfft.SLAB_Z_THEN_YX
    kinds = tuple(KIND[n] for n in names)
    xg = np.random.default_rng(5).standard_normal(shape)
    ref = global_ref(xg, kinds, False, 3)
    isz, ist = dfft.layout(dec, dfft.DCT, *shape, p1, p2, rank, 0)
    osz, ost = dfft.layout(dec, dfft.DCT, *shape, p1, p2, rank, 3)
    dt = torch.float64 if f64 else torch.float32
    x = torch.from_numpy(np.ascontiguousarray(blk(xg, isz, ist))).to("cuda", dt)
    spec = torch.empty(plan.getDomainSize() // (8 if f64 else 4), dtype=dt, device="cuda")
    back = torch.empty_like(x)
    plan.execR2R(spec, x, dfft.FORWARD)
    n_out = osz[0] * osz[1] * osz[2]
    tol = 1e-10 if f64 else 1e-5
    ok = rel(spec[:n_out].reshape(osz).cpu().double().numpy(), blk(ref, osz, ost)) < tol
    plan.execR2R(back, spec, dfft.INVERSE)
    factor = float(np.prod([(n + N_OF.get(k, 0)) * PER_AXIS[k] for n, k in zip(shape, names)]))
    ok &= rel(back.cpu().double().numpy() / factor, blk(xg, isz, ist)) < tol
    plan.destroy()
    t = torch.tensor([0.0 if ok else 1.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item() == 0


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = dfft.Comm.from_torch_distributed(local)
    fails = 0
    for shape in ((32, 64, 128), (16, 32, 16 * world)):
        for decomp in ("slab", "zyx", "pencil"):
            for names in (("dct4", "r2hc", "r2hc"), ("dst4", "dst4", "dst4"), ("dct4", "dst", "dst1"), ("dct4", "dst4", "r2hc")):
                for comm_method in (P2P, A2A):
                    for send in (SYNC, STREAMS):
                        for f64 in (True, False):
                            ok = check(comm, world, rank, decomp, names, comm_method, send, f64, shape)
                            if rank == 0:
                                print(f"{'ok  ' if ok else 'FAIL'} {shape} {decomp} {names} {comm_method.name} {send.name} {'f64' if f64 else 'f32'}",
                                      flush=True)
                            fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_r2r4: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
