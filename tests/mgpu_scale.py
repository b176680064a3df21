"""Output scale on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_scale.py

For slab and pencil plans, Peer2Peer and All2All, Sync and tuned Streams schedules, forward and inverse, every rank's
scaled output must equal its unscaled output of the same plan times the scale, bit for bit (torch, same dtype)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
SYNC, STREAMS = dfft.SendMethod.Sync, dfft.SendMethod.Streams


def bits(t):
    r = torch.view_as_real(t) if t.is_complex() else t
    return r.contiguous().view(torch.int64 if r.dtype == torch.float64 else torch.int32)


def check(comm, world, decomp, transform, comm_method, send, shape=(64, 64, 128), scale=0.3):
    cfg = dfft.Configurations(comm_method=comm_method, send_method=send, comm_method2=comm_method, send_method2=send)
    if decomp == "slab":
        plan = dfft.MPIcuFFT_Slab(cfg, comm, precision="double", transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), None, True)
    else:
        p1 = 2 if world % 2 == 0 else 1
        plan = dfft.MPIcuFFT_Pencil(cfg, comm, precision="double", transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, world // p1), True)
    c2c = transform == "c2c"
    isz = plan.getInSize()
    n_in = isz[0] * isz[1] * isz[2]
    g = torch.Generator(device="cuda").manual_seed(11 + dist.get_rank())
    real = torch.rand(n_in, generator=g, device="cuda", dtype=torch.float64)
    x = torch.complex(real, torch.rand(n_in, generator=g, device="cuda", dtype=torch.float64)) if c2c else real
    spec = torch.empty(plan.getDomainSize() // 16, dtype=torch.complex128, device="cuda")
    back = torch.empty_like(x)

    def fwd():
        plan.execC2C(spec, x, dfft.FORWARD) if c2c else plan.execR2C(spec, x)

    def inv():
        plan.execC2C(back, spec, dfft.INVERSE) if c2c else plan.execC2R(back, spec)

    if send == STREAMS:
        plan.tune(spec, x, dfft.FORWARD)
        plan.tune(back, spec, dfft.INVERSE) if c2c else None
    ok = True
    osz = plan.getOutSize()
    n_out = osz[0] * osz[1] * osz[2]
    fwd()
    ref_spec = spec[:n_out].clone()
    plan.setScale(scale, 1.0)
    fwd()
    ok &= torch.equal(bits(spec[:n_out]), bits(torch.view_as_real(ref_spec) * scale))
    plan.setScale(1.0, 1.0)
    fwd()
    inv()
    ref_back = back.clone()
    plan.setScale(1.0, scale)
    inv()
    want = (torch.view_as_real(ref_back) if c2c else ref_back) * scale
    ok &= torch.equal(bits(back), bits(want))
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
    for decomp in ("slab", "pencil"):
        for transform in ("c2c", "r2c"):
            for comm_method in (P2P, A2A):
                for send in (SYNC, STREAMS):
                    ok = check(comm, world, decomp, transform, comm_method, send)
                    if rank == 0:
                        print(f"{'ok  ' if ok else 'FAIL'} {decomp} {transform} {comm_method.name} {send.name}", flush=True)
                    fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_scale: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
