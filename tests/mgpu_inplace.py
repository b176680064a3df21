"""In-place plans on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_inplace.py

For slab and pencil plans, C2C and R2C, Peer2Peer and All2All, Sync and Streams schedules (the overlapped ones included),
forward and inverse, batch 1 and 2: every rank's in-place output must equal the out-of-place plan's output on the same
input bit for bit.  The in-place buffer holds getDomainSize() bytes per field; R2C rows are padded to Nz/2 + 1 complex."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
SYNC, STREAMS = dfft.SendMethod.Sync, dfft.SendMethod.Streams


def make(comm, world, decomp, transform, cfg, shape, batch, inplace):
    if decomp == "slab":
        plan = dfft.MPIcuFFT_Slab(cfg, comm, precision="double", transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), None, True, batch, inplace)
    else:
        p1 = 2 if world % 2 == 0 else 1
        plan = dfft.MPIcuFFT_Pencil(cfg, comm, precision="double", transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, world // p1), True, batch, inplace)
    return plan


def check(comm, world, decomp, transform, comm_method, send, batch, shape=(64, 48, 128)):
    cfg = dfft.Configurations(comm_method=comm_method, send_method=send, comm_method2=comm_method, send_method2=send)
    oop = make(comm, world, decomp, transform, cfg, shape, batch, False)
    ip = make(comm, world, decomp, transform, cfg, shape, batch, True)
    c2c = transform == "c2c"
    isz, osz = oop.getInSize(), oop.getOutSize()
    n_in, n_out = isz[0] * isz[1] * isz[2], osz[0] * osz[1] * osz[2]
    dom = ip.getDomainSize() // 16
    nz, nzc = shape[2], shape[2] // 2 + 1
    g = torch.Generator(device="cuda").manual_seed(5 + dist.get_rank())
    real = torch.rand((batch, n_in), generator=g, device="cuda", dtype=torch.float64)
    x = torch.complex(real, torch.rand((batch, n_in), generator=g, device="cuda", dtype=torch.float64)) if c2c else real
    spec = torch.empty((batch, n_out), dtype=torch.complex128, device="cuda")
    back = torch.empty_like(x)
    buf = torch.empty((batch, dom), dtype=torch.complex128, device="cuda")

    def real_side(f):  # C2C: plain; R2C: padded rows, the first Nz reals of every row
        if c2c:
            return buf[f, :n_in]
        return torch.view_as_real(buf[f, :isz[0] * isz[1] * nzc]).reshape(isz[0] * isz[1], 2 * nzc)[:, :nz]

    def run(plan, out, in_, inverse):
        if c2c:
            plan.execC2C(out, in_, dfft.INVERSE if inverse else dfft.FORWARD)
        else:
            plan.execC2R(out, in_) if inverse else plan.execR2C(out, in_)

    if send == STREAMS:  # the same candidates for both plans; each keeps its own winner
        for p_, o_, i_ in ((oop, spec, x), (ip, buf, buf)):
            p_.tune(o_, i_, dfft.FORWARD)
    ok = True
    run(oop, spec, x, 0)
    for f in range(batch):
        real_side(f).copy_(x[f].reshape(real_side(f).shape))
    run(ip, buf, buf, 0)
    ok &= torch.equal(buf[:, :n_out], spec)
    run(oop, back, spec, 1)
    buf[:, :n_out] = spec
    run(ip, buf, buf, 1)
    for f in range(batch):
        ok &= torch.equal(real_side(f), back[f].reshape(real_side(f).shape))
    oop.destroy()
    ip.destroy()
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
                    for batch in (1, 2):
                        ok = check(comm, world, decomp, transform, comm_method, send, batch)
                        if rank == 0:
                            print(f"{'ok  ' if ok else 'FAIL'} {decomp} {transform} {comm_method.name} {send.name} batch {batch}", flush=True)
                        fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_inplace: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
