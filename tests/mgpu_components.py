"""Interleaved multi-component plans on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_components.py

For slab ZY_Then_X, Z_Then_YX and pencil plans, Peer2Peer and All2All, C2C and R2C / C2R, f64, odd and even C: every rank's
block of the forward must match numpy's fftn / rfftn over axes 0-2 of the global [X, Y, Z, C] array, and its block of the
inverse the unnormalised inverse of the global spectrum, to 1e-10."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def check(comm, world, decomp, transform, comm_method, comps, shape=(32, 64, 128)):
    cfg = dfft.Configurations(comm_method=comm_method, comm_method2=comm_method)
    plan = CLASSES[decomp](cfg, comm, precision="double", transform=transform)
    p1 = 2 if world % 2 == 0 else 1
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, world // p1) if decomp == "pencil" else None, True, components=comps)
    c2c = transform == "c2c"
    rng = np.random.default_rng(7)
    g = shape + (comps,)
    x = rng.standard_normal(g) + (1j * rng.standard_normal(g) if c2c else 0)
    X = np.fft.fftn(x, axes=(0, 1, 2)) if c2c else np.fft.rfftn(x, axes=(0, 1, 2))
    n = shape[0] * shape[1] * shape[2]
    y = x * n
    isz, ist, osz, ost = plan.getInSize(), plan.getInStart(), plan.getOutSize(), plan.getOutStart()
    blk = lambda a, s, o: np.ascontiguousarray(a[o[0]:o[0] + s[0], o[1]:o[1] + s[1], o[2]:o[2] + s[2]])
    xin = torch.from_numpy(blk(x, isz, ist)).cuda()
    out = torch.empty(tuple(osz) + (comps,), dtype=torch.complex128, device="cuda")
    plan.execC2C(out, xin, dfft.FORWARD) if c2c else plan.execR2C(out, xin)
    ok = rel(out.cpu().numpy(), blk(X, osz, ost)) < 1e-10
    back = torch.empty_like(xin)
    Xin = torch.from_numpy(blk(X, osz, ost)).cuda()
    plan.execC2C(back, Xin, dfft.INVERSE) if c2c else plan.execC2R(back, Xin)
    ok &= rel(back.cpu().numpy(), blk(y, isz, ist)) < 1e-10
    plan.destroy()
    r = torch.tensor([0.0 if ok else 1.0], device="cuda")
    dist.all_reduce(r, op=dist.ReduceOp.MAX)
    return r.item() == 0


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = dfft.Comm.from_torch_distributed(local)
    fails = 0
    for decomp in ("slab", "zyx", "pencil"):
        for transform in ("c2c", "r2c"):
            for comm_method in (P2P, A2A):
                for comps in (2, 3):
                    ok = check(comm, world, decomp, transform, comm_method, comps)
                    if rank == 0:
                        print(f"{'ok  ' if ok else 'FAIL'} {decomp} {transform} {comm_method.name} C={comps}", flush=True)
                    fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_components: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
