"""16-bit plans on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_half.py

For slab ZY_Then_X and pencil plans, Peer2Peer and All2All, C2C and R2C / C2R, FP16 and BF16, scales (1/sqrt(N),
1/sqrt(N)): every rank's block of the forward must match the float64 transform of the widened global input over sqrt(N),
and its block of the inverse of that spectrum the widened input, within the bounds of tests/test_gpu_half.py (rel-L2
2e-3 FP16, 1.6e-2 BF16)."""
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "pencil": dfft.MPIcuFFT_Pencil}
DTYPE = {"half": torch.float16, "bfloat16": torch.bfloat16}
TOL = {"half": 2e-3, "bfloat16": 1.6e-2}


def rel(a, b):
    return float(torch.linalg.vector_norm(a - b) / torch.linalg.vector_norm(b))


def block(a, s, o):
    return a[o[0]:o[0] + s[0], o[1]:o[1] + s[1], o[2]:o[2] + s[2]].contiguous()


def check(comm, world, decomp, transform, comm_method, prec, shape=(64, 128, 256)):
    cfg = dfft.Configurations(comm_method=comm_method, comm_method2=comm_method)
    plan = CLASSES[decomp](cfg, comm, precision=prec, transform=transform)
    p1 = 2 if world % 2 == 0 else 1
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, world // p1) if decomp == "pencil" else None, True)
    N = shape[0] * shape[1] * shape[2]
    plan.setScale(N ** -0.5, N ** -0.5)  # the normalisation recommended for FP16
    c2c = transform == "c2c"
    g = torch.Generator(device="cuda").manual_seed(5)  # the same global field on every rank
    x16 = (torch.randn(shape + ((2,) if c2c else ()), generator=g, device="cuda") * 0.25).to(DTYPE[prec])
    xd = torch.view_as_complex(x16.double()) if c2c else x16.double()
    X = torch.fft.fftn(xd) if c2c else torch.fft.rfftn(xd)
    isz, ist, osz, ost = plan.getInSize(), plan.getInStart(), plan.getOutSize(), plan.getOutStart()
    xin = block(x16, isz, ist)
    out = torch.empty(tuple(osz) + (2,), dtype=DTYPE[prec], device="cuda")
    plan.execC2C(out, xin, dfft.FORWARD) if c2c else plan.execR2C(out, xin)
    ok = rel(torch.view_as_complex(out.double()), block(X * N ** -0.5, osz, ost)) < TOL[prec]
    # inverse of the spectrum X / sqrt(N), scaled by 1 / sqrt(N): the input again
    spec = block(torch.view_as_real(X * N ** -0.5).to(DTYPE[prec]), osz, ost)
    back = torch.empty_like(xin)
    plan.execC2C(back, spec, dfft.INVERSE) if c2c else plan.execC2R(back, spec)
    got = torch.view_as_complex(back.double()) if c2c else back.double()
    ok &= rel(got, block(xd, isz, ist)) < TOL[prec]
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
    for decomp in ("slab", "pencil"):
        for transform in ("c2c", "r2c"):
            for comm_method in (P2P, A2A):
                for prec in ("half", "bfloat16"):
                    ok = check(comm, world, decomp, transform, comm_method, prec)
                    if rank == 0:
                        print(f"{'ok  ' if ok else 'FAIL'} {decomp} {transform} {comm_method.name} {prec}", flush=True)
                    fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_half: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
