"""Box-distributed plans on several GPUs (run under torchrun with 2-8 GPUs):

    torchrun --nproc-per-node N tests/mgpu_boxes.py

For slab, Z_Then_YX and pencil plans, Peer2Peer and All2All, C2C, R2C / C2R and DCT, f64 and f32: every rank regenerates
the seeded global array, passes its brick of it (bricks of a Px x Py x Pz grid of the rank count, uneven on odd counts),
compares its output brick with numpy's transform of the whole array, then checks that the inverse returns its input brick
times the grid size.  The redistribution runs through peer memory or NCCL between real processes, which the one-GPU
replays of tests/test_gpu_boxes.py do not exercise."""
import os
import sys

import numpy as np
import scipy.fft as sf
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import distributedfft_b200 as dfft  # noqa: E402

P2P, A2A = dfft.CommunicationMethod.Peer2Peer, dfft.CommunicationMethod.All2All


def grid_of(P):
    """Px x Py x Pz with Px * Py * Pz = P, as cubic as it goes"""
    best = None
    for px in range(1, P + 1):
        for py in range(1, P // px + 1):
            if P % (px * py) == 0:
                g = (px, py, P // (px * py))
                if best is None or max(g) < max(best):
                    best = g
    return best


def bricks(shape, parts):
    cuts = [[i * shape[a] // parts[a] // 2 * 2 if a == 2 else i * shape[a] // parts[a] for i in range(parts[a] + 1)] for a in range(3)]
    for a in range(3):
        cuts[a][-1] = shape[a]
    return [((cuts[0][i], cuts[1][j], cuts[2][k]), (cuts[0][i + 1], cuts[1][j + 1], cuts[2][k + 1]))
            for i in range(parts[0]) for j in range(parts[1]) for k in range(parts[2])]


def blk(a, box):
    (l0, l1, l2), (h0, h1, h2) = box
    return a[l0:h0, l1:h1, l2:h2]


def check(comm, world, rank, decomp, transform, comm_method, f64, shape):
    cfg = dfft.Configurations(comm_method=comm_method, comm_method2=comm_method)
    prec = "double" if f64 else "float"
    parts = grid_of(world)
    ib = bricks(shape, parts)
    nzc = shape[2] // 2 + 1 if transform == "r2c" else shape[2]
    ob = bricks((shape[0], shape[1], nzc), parts[::-1])
    if decomp == "pencil":
        p1 = 2 if world % 2 == 0 else 1
        plan = dfft.MPIcuFFT_Pencil(cfg, comm, precision=prec, transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(p1, world // p1), True, in_boxes=ib, out_boxes=ob)
    else:
        cls = dfft.MPIcuFFT_Slab if decomp == "slab" else dfft.MPIcuFFT_Slab_Z_Then_YX
        plan = cls(cfg, comm, precision=prec, transform=transform)
        plan.initFFT(dfft.GlobalSize(*shape), None, True, in_boxes=ib, out_boxes=ob)
    rng = np.random.default_rng(7)
    real = transform != "c2c"
    xg = rng.standard_normal(shape) if real else rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    if transform == "c2c":
        ref, factor = np.fft.fftn(xg), np.prod(shape)
    elif transform == "r2c":
        ref, factor = np.fft.rfftn(xg), np.prod(shape)
    else:
        ref, factor = sf.dctn(xg, type=2), 8 * np.prod(shape)
    rdt, cdt = (torch.float64, torch.complex128) if f64 else (torch.float32, torch.complex64)
    x = torch.from_numpy(np.ascontiguousarray(blk(xg, ib[rank]))).to("cuda", rdt if real else cdt)
    osz = [h - l for l, h in zip(*ob[rank])]
    spec = torch.empty(osz, dtype=rdt if transform == "dct" else cdt, device="cuda")
    back = torch.empty_like(x)
    if transform == "c2c":
        plan.execC2C(spec, x, dfft.FORWARD); fwd = spec.cpu().numpy()
        plan.execC2C(back, spec, dfft.INVERSE)
    elif transform == "r2c":
        plan.execR2C(spec, x); fwd = spec.cpu().numpy()
        plan.execC2R(back, spec)
    else:
        plan.execR2R(spec, x, dfft.FORWARD); fwd = spec.cpu().numpy()
        plan.execR2R(back, spec, dfft.INVERSE)
    tol = 1e-10 if f64 else 1e-4
    want = blk(ref, ob[rank])
    ok = np.linalg.norm(fwd - want) <= tol * np.linalg.norm(want)
    want = blk(xg, ib[rank])
    ok &= np.linalg.norm(back.cpu().numpy() / factor - want) <= tol * np.linalg.norm(want)
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
    for shape in ((32, 64, 128), (16 * world, 32, 64)):
        for decomp in ("slab", "zyx", "pencil"):
            for transform in ("c2c", "r2c", "dct"):
                for comm_method in (P2P, A2A):
                    for f64 in (True, False):
                        ok = check(comm, world, rank, decomp, transform, comm_method, f64, shape)
                        if rank == 0:
                            print(f"{'ok  ' if ok else 'FAIL'} {shape} {decomp} {transform} {comm_method.name} {'f64' if f64 else 'f32'}", flush=True)
                        fails += 0 if ok else 1
    if rank == 0:
        print(f"mgpu_boxes: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
