"""Capture of multi-rank plans is refused (run under torchrun with two or more GPUs):

    torchrun --nproc-per-node N tests/mgpu_graph_capture.py

On every rank an `_async` exec on a capturing stream returns DFFT_ERR_UNSUPPORTED, and the plan then
runs eagerly and matches the oracle as before."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402
from distributedfft_b200._lib import DfftError  # noqa: E402
from oracle import dft_oracle as O  # noqa: E402

DFFT_ERR_UNSUPPORTED = -5  # include/dfft.h


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = dfft.Comm.from_torch_distributed(local)
    shape = (64, 64, 64)
    fails = 0
    for cls, grid in ((dfft.MPIcuFFT_Slab, None), (dfft.MPIcuFFT_Pencil, (1, world))):
        plan = cls(dfft.Configurations(), comm, precision="double", transform="c2c")
        plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(*grid) if grid else None, True)
        isz, ist, osz, ost = plan.getInSize(), plan.getInStart(), plan.getOutSize(), plan.getOutStart()
        xg = O.complex_input(shape)
        xin = torch.from_numpy(np.ascontiguousarray(O.block(xg, ist, isz))).cuda()
        out = torch.empty(plan.getDomainSize() // 16, dtype=torch.complex128, device="cuda")
        s = torch.cuda.current_stream()
        plan.execC2C(out, xin, dfft.FORWARD, stream=s)  # warmed up: the refusal is about the rank count alone
        plan.wait()
        code = 0
        g = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(g):
                plan.execC2C(out, xin, dfft.FORWARD, stream=torch.cuda.current_stream())
        except DfftError as e:
            code = e.code
        del g
        out.zero_()
        plan.execC2C(out, xin, dfft.FORWARD, stream=s)
        plan.wait()
        n_out = osz[0] * osz[1] * osz[2]
        err = O.rel_l2(out[:n_out].cpu().numpy().reshape(osz), O.block(O.fft_c2c(xg), ost, osz))
        ok = code == DFFT_ERR_UNSUPPORTED and err < 1e-10
        t = torch.tensor([0.0 if ok else 1.0], device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(f"{'ok  ' if t.item() == 0 else 'FAIL'} {cls.__name__}: capture -> {code}, eager exec after it rel-L2 {err:.2e}", flush=True)
        fails += int(t.item())
        plan.destroy()
    if rank == 0:
        print(f"mgpu_graph_capture: {fails} failed", flush=True)
    comm.destroy()
    dist.destroy_process_group()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
