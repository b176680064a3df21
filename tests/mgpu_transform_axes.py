"""Plans with kept (untransformed) axes on several GPUs (run under torchrun with 2-8 GPUs):

    torchrun --nproc-per-node N tests/mgpu_transform_axes.py

For slab, Z_Then_YX and pencil plans, Peer2Peer and All2All, Sync and Streams (which runs the sequential schedule for these
plans), every mask of C2C plans, x kept on mixed R2R plans and f64 / f32: every rank regenerates the seeded global array,
compares its own block of the forward output with the transform of the whole array over the transformed axes only, then
checks the inverse through the round trip of its block, which scales by the product of the transformed lengths."""
import itertools
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import distributedfft_b200 as dfft  # noqa: E402
from test_r2r_mixed import r2r_1d  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
SYNC, STREAMS = dfft.SendMethod.Sync, dfft.SendMethod.Streams
KIND = {"dct": dfft.DCT, "dst": dfft.DST, "r2hc": dfft.R2HC}


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def blk(a, size, start):
    return a[start[0]:start[0] + size[0], start[1]:start[1] + size[1], start[2]:start[2] + size[2]]


def check(comm, world, rank, decomp, transform, axes, comm_method, send, f64, shape):
    cfg = dfft.Configurations(comm_method=comm_method, send_method=send, comm_method2=comm_method, send_method2=send)
    prec = "double" if f64 else "float"
    real = isinstance(transform, tuple)
    if decomp == "pencil":
        p1 = 2 if world % 2 == 0 else 1
        p2 = world // p1
        plan = dfft.MPIcuFFT_Pencil(cfg, comm, precision=prec, transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, p2), True, transform_axes=axes)
        dec = dfft.PENCIL
    else:
        p1, p2 = world, 1
        cls = dfft.MPIcuFFT_Slab if decomp == "slab" else dfft.MPIcuFFT_Slab_Z_Then_YX
        plan = cls(cfg, comm, precision=prec, transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), None, True, transform_axes=axes)
        dec = dfft.SLAB_ZY_THEN_X if decomp == "slab" else dfft.SLAB_Z_THEN_YX
    rng = np.random.default_rng(5)
    xg = rng.standard_normal(shape) if real else rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    ref, factor = xg, 1.0
    for a in (2, 1, 0):
        if axes[a]:
            ref = r2r_1d(ref, KIND[transform[a]], False, a) if real else np.fft.fft(ref, axis=a)
            factor *= shape[a] * (2 if real and transform[a] != "r2hc" else 1)
    lay_t = dfft.DCT if real else dfft.C2C
    isz, ist = dfft.layout(dec, lay_t, *shape, p1, p2, rank, 0)
    osz, ost = dfft.layout(dec, lay_t, *shape, p1, p2, rank, 3)
    dt = (torch.float64 if f64 else torch.float32) if real else (torch.complex128 if f64 else torch.complex64)
    x = torch.from_numpy(np.ascontiguousarray(blk(xg, isz, ist))).to("cuda", dt)
    spec = torch.empty(max(plan.getDomainSize() // x.element_size(), 1), dtype=dt, device="cuda")
    back = torch.empty_like(x)
    ex = plan.execR2R if real else plan.execC2C
    ex(spec, x, dfft.FORWARD)
    n_out = osz[0] * osz[1] * osz[2]
    tol = 1e-10 if f64 else 1e-5
    ok = rel(spec[:n_out].reshape(osz).cpu().numpy().astype(xg.dtype), blk(ref, osz, ost)) < tol
    ex(back, spec, dfft.INVERSE)
    ok &= rel(back.cpu().numpy().astype(xg.dtype) / factor, blk(xg, isz, ist)) < tol
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
    cases = [("c2c", axes) for axes in itertools.product((False, True), repeat=3)]
    cases += [(("dct", "r2hc", "r2hc"), (False, True, True)), (("dst", "r2hc", "dct"), (False, True, True))]
    for shape in ((32, 64, 128), (16 * world, 24, 20)):
        for decomp in ("slab", "zyx", "pencil"):
            for transform, axes in cases:
                for comm_method in (P2P, A2A):
                    for send in (SYNC, STREAMS):
                        for f64 in (True, False):
                            if isinstance(transform, tuple) and shape[1] == 24:
                                continue  # real-to-real plans take powers of two
                            ok = check(comm, world, rank, decomp, transform, axes, comm_method, send, f64, shape)
                            if rank == 0:
                                print(f"{'ok  ' if ok else 'FAIL'} {shape} {decomp} {transform} {axes} {comm_method.name} {send.name} "
                                      f"{'f64' if f64 else 'f32'}", flush=True)
                            fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_transform_axes: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
