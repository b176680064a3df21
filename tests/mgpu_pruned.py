"""Pruned plans on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_pruned.py

For slab ZY_Then_X, Z_Then_YX and pencil plans, Peer2Peer and All2All, C2C and R2C / C2R, f64: every rank's block of the
forward of a field whose data block is smaller than the transform grid must match numpy's fftn / rfftn of the zero-embedded
field through the index map (tests/test_pruned.py), and its block of the inverse the unnormalised inverse truncated to the
data block, to 1e-10."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import distributedfft_b200 as dfft  # noqa: E402
from test_pruned import fwd_ref, inv_ref  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def check(comm, world, decomp, transform, comm_method, shape=(32, 64, 128), data=(16, 33, 66), spec=(21, 43, 85)):
    cfg = dfft.Configurations(comm_method=comm_method, comm_method2=comm_method)
    plan = CLASSES[decomp](cfg, comm, precision="double", transform=transform)
    p1 = 2 if world % 2 == 0 else 1
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, world // p1) if decomp == "pencil" else None, True, spectral=spec, data=data)
    c2c = transform == "c2c"
    t = dfft.C2C if c2c else dfft.R2C
    rng = np.random.default_rng(5)
    x = rng.standard_normal(data) + (1j * rng.standard_normal(data) if c2c else 0)
    X = fwd_ref(x, t, shape, spec, 3)
    y = inv_ref(X, t, shape, data, spec, 3)
    y = y if c2c else y.real
    isz, ist, osz, ost = plan.getInSize(), plan.getInStart(), plan.getOutSize(), plan.getOutStart()
    blk = lambda a, s, o: np.ascontiguousarray(a[o[0]:o[0] + s[0], o[1]:o[1] + s[1], o[2]:o[2] + s[2]])
    xin = torch.from_numpy(blk(x, isz, ist)).cuda()
    out = torch.empty(tuple(osz), dtype=torch.complex128, device="cuda")
    plan.execC2C(out, xin, dfft.FORWARD) if c2c else plan.execR2C(out, xin)
    ok = rel(out.cpu().numpy(), blk(X, osz, ost)) < 1e-10
    back = torch.empty_like(xin)
    plan.execC2C(back, torch.from_numpy(blk(X, osz, ost)).cuda(), dfft.INVERSE) if c2c else plan.execC2R(back, torch.from_numpy(blk(X, osz, ost)).cuda())
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
                ok = check(comm, world, decomp, transform, comm_method)
                if rank == 0:
                    print(f"{'ok  ' if ok else 'FAIL'} {decomp} {transform} {comm_method.name}", flush=True)
                fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_pruned: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
