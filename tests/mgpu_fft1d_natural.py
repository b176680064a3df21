"""Natural-order distributed 1D transforms on several GPUs (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_fft1d_natural.py

For Peer2Peer and All2All, f64 and f32, default and explicit factors: every rank transforms its chunk of one seeded signal;
each rank's output chunk must match its contiguous slice of torch.fft.fft of the whole signal, the gathered chunks must
tile the spectrum in rank order (rel-L2 < 1e-12 / 1e-5), and the inverse must return n times each rank's input chunk."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All


def rel(got, want):
    return float(torch.linalg.vector_norm(got - want) / torch.linalg.vector_norm(want))


def check(comm, world, comm_method, precision, n, factors):
    cdt = torch.complex128 if precision == "double" else torch.complex64
    bound = 1e-12 if precision == "double" else 1e-5
    cfg = dfft.Configurations(comm_method=comm_method, comm_method2=comm_method)
    plan = dfft.MPIcuFFT_Slab(cfg, comm, precision=precision, transform="c2c")
    plan.initFFT(None, signal=n, factors=factors, natural=True)
    n1, n2, n3 = plan.getFactors()
    rows, start = plan.getInSize()[0], plan.getInStart()[0]
    planes, k3 = plan.getOutSize()[0], plan.getOutStart()[0]
    g = torch.Generator(device="cuda").manual_seed(1234)
    whole = torch.randn(n, dtype=cdt, device="cuda", generator=g)  # the same signal on every rank
    chunk = whole[start * n2 * n3:(start + rows) * n2 * n3].view(rows, n2, n3).clone()
    spec = torch.empty((planes, n2, n1), dtype=cdt, device="cuda")
    plan.execC2C(spec, chunk, dfft.FORWARD)
    want = torch.fft.fft(whole)
    lo, hi = k3 * n1 * n2, (k3 + planes) * n1 * n2
    err = rel(spec.reshape(-1), want[lo:hi])  # my slice of the spectrum, no index map
    parts = [None] * world
    dist.all_gather_object(parts, (lo, hi, spec.cpu()))
    full = torch.cat([p for _, _, p in sorted(parts, key=lambda t: t[0])]).reshape(-1)
    tiled = [(a, b) for a, b, _ in sorted(parts, key=lambda t: t[0])]
    tiles = tiled[0][0] == 0 and tiled[-1][1] == n and all(b == c for (_, b), (c, _) in zip(tiled, tiled[1:]))
    err_all = rel(full, want.cpu())
    back = torch.empty_like(chunk)
    plan.execC2C(back, spec, dfft.INVERSE)
    err_b = rel(back, n * chunk)
    plan.destroy()
    return tiles and max(err, err_all) < bound and err_b < bound, max(err, err_all), err_b


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = dfft.Comm.from_torch_distributed(local)
    fails = 0
    for comm_method in (P2P, A2A):
        for precision in ("double", "float"):
            for n, factors in ((1 << 20, None), (1 << 24, None), (1 << 18, (64, 64, 64))):
                ok, err, err_b = check(comm, world, comm_method, precision, n, factors)
                if rank == 0:
                    print(f"{'ok  ' if ok else 'FAIL'} {comm_method.name} {precision} n=2^{n.bit_length() - 1} factors={factors}: "
                          f"forward {err:.2e} round trip {err_b:.2e}", flush=True)
                fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_fft1d_natural: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
