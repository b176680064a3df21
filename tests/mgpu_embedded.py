"""Plans with strides (dfft_plan_set_strides) on several GPUs (run under torchrun with 2-8 GPUs):

    torchrun --nproc-per-node N tests/mgpu_embedded.py

For slab, Z_Then_YX and pencil plans, Peer2Peer and All2All, C2C, R2C / C2R and DCT, f64: every rank regenerates the
seeded global array, holds its input block as the interior of an array with two ghost layers per side (NaN) and its output
block the same way, runs the forward exec on the interiors and compares its output block bit for bit with the same plan
without strides on dense tensors, then runs the inverse back into the input array's interior and compares again.  Every
ghost element must still be NaN and the input array unchanged.  The peer stores and NCCL exchanges between real processes
are what the one-GPU replays of tests/test_gpu_embedded.py do not exercise."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All
H = 2
CLS = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}


def halo(size, dtype):
    a = torch.full([n + 2 * H for n in size], float("nan"), dtype=dtype, device="cuda")
    return a, a[H:-H, H:-H, H:-H]


def strides(t):
    return (t.shape[0] * t.stride(0),) + tuple(t.stride()[:2])


def same(a, b):
    return torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def make(decomp, transform, comm, method, P, in_strides=None, out_strides=None):
    cfg = dfft.Configurations(comm_method=method, comm_method2=method)
    f = CLS[decomp](cfg, comm, precision="double", transform=transform)
    part = None
    if decomp == "pencil":
        p1 = max(d for d in range(1, int(P ** 0.5) + 1) if P % d == 0)
        part = dfft.Partition(p1, P // p1)
    f.initFFT(dfft.GlobalSize(16, 16, 32), part, True, in_strides=in_strides, out_strides=out_strides)
    return f


def run(decomp, transform, method, comm, P, rank):
    kind = {"c2c": "c2c", "r2c": "r2c", "dct": "r2r"}[transform]
    plain = make(decomp, transform, comm, method, P)
    phys_t = torch.complex128 if kind == "c2c" else torch.float64
    spec_t = torch.float64 if kind == "r2r" else torch.complex128
    a_in, phys = halo(plain.getInSize(), phys_t)
    a_out, spec = halo(plain.getOutSize(), spec_t)
    f = make(decomp, transform, comm, method, P, strides(phys), strides(spec))
    rng = np.random.default_rng(7)
    g = rng.standard_normal((16, 16, 32)) + (1j * rng.standard_normal((16, 16, 32)) if kind == "c2c" else 0)
    (s0, s1, s2), (n0, n1, n2) = plain.getInStart(), plain.getInSize()
    x = torch.from_numpy(np.ascontiguousarray(g[s0:s0 + n0, s1:s1 + n1, s2:s2 + n2])).cuda()
    phys.copy_(x)

    def exe(p, out, in_, inverse):
        if kind == "c2c":
            p.execC2C(out, in_, dfft.INVERSE if inverse else dfft.FORWARD)
        elif kind == "r2c":
            (p.execC2R if inverse else p.execR2C)(out, in_)
        else:
            p.execR2R(out, in_, dfft.INVERSE if inverse else dfft.FORWARD)

    want = torch.empty(plain.getOutSize(), dtype=spec_t, device="cuda")
    exe(plain, want, x, False)
    before = a_in.clone()
    exe(f, spec, phys, False)
    ok = same(spec, want) and same(a_in, before)
    back = torch.empty_like(x)
    exe(plain, back, want, True)
    exe(f, phys, spec, True)
    ok = ok and same(phys, back)
    for a in (a_in, a_out):
        ghost = torch.ones_like(a, dtype=torch.bool)
        ghost[H:-H, H:-H, H:-H] = False
        ok = ok and bool(torch.isnan(a[ghost]).all())
    f.destroy()
    plain.destroy()
    return ok


def main():
    dist.init_process_group("gloo")
    rank, P = dist.get_rank(), dist.get_world_size()
    torch.cuda.set_device(rank % torch.cuda.device_count())
    comm = dfft.Comm.from_torch_distributed()
    failures = 0
    for decomp in ("slab", "zyx", "pencil"):
        for transform in ("c2c", "r2c", "dct"):
            for method, mname in ((P2P, "p2p"), (A2A, "a2a")):
                ok = run(decomp, transform, method, comm, P, rank)
                flag = torch.tensor([0 if ok else 1])
                dist.all_reduce(flag)
                failures += int(flag.item())
                if rank == 0:
                    print(f"{decomp} {transform} {mname}: {'ok' if flag.item() == 0 else 'FAILED'}", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    if rank == 0:
        print("PASSED" if failures == 0 else f"FAILED ({failures})")
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
