"""Pruned plans against the caller's own zero-embedding on one GPU.

A 512^3 transform grid with a 256^3 field (the doubled grid of a free-space solve), f64 and f32, C2C and R2C / C2R. It times
  * the pruned plan's forward and inverse (dfft_plan_create_pruned), and their passes from the step timer;
  * the ordinary 512^3 plan with the caller's torch work: zero-fill and copy-in before the forward, slice-out after the
    inverse;
  * the HBM-byte floor of each at 3.35 TB/s (the H100 SXM data sheet), from the bytes every pass must read and write
    (the ordinary one-rank C2C plan runs the fused z + y stage: two sweeps over the grid instead of three).
The two paths run in alternating windows of CUDA-event-timed execs, and the card's name, power limit and max SM clock are
read in the same run.  It also reports whether the pruned forward spectrum equals the embedded one bit for bit, and the
work area (dfft_get_work_size_device) of both plans.  A report, not a gate: it prints one JSON line per case (and writes
them to --out).

    python tools/pruned_bench.py [--n 512] [--m 256] [--reps 20] [--windows 5] [--out pruned_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def floors(n, m, es, r2c):
    """least HBM bytes of the forward and of the inverse of each path: every pass reads and writes its arrays once"""
    nzc = n // 2 + 1 if r2c else n
    real = es // 2 if r2c else es  # the physical side of R2C is real
    phys_n, phys_m = n * n * n * real, m * m * m * real
    grid = n * n * nzc * es
    pruned = phys_m + (2 * m * m * nzc + 2 * m * n * nzc) * es + grid  # z, y, x passes
    sweeps = 3 if r2c else 2  # the fused z + y stage of one-rank C2C plans reads and writes the grid once
    ordinary = phys_n + grid + (2 * sweeps - 2) * grid
    embed = phys_n + 2 * phys_m  # zero-fill the grid, copy the field in
    slice_out = 2 * phys_m
    return {"pruned_fwd": pruned, "ordinary_fwd": ordinary + embed, "pruned_inv": pruned, "ordinary_inv": ordinary + slice_out}


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--m", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20, help="execs per timed window")
    ap.add_argument("--windows", type=int, default=5, help="alternating windows per path")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import distributedfft_b200 as dfft

    if not torch.cuda.is_available():
        raise SystemExit("pruned_bench.py needs a CUDA device")
    n, m = args.n, args.m
    dev = "cuda"
    info = card()
    results = []
    for prec in ("double", "float"):
        for transform in ("c2c", "r2c"):
            r2c = transform == "r2c"
            cdt = torch.complex128 if prec == "double" else torch.complex64
            rdt = torch.float64 if prec == "double" else torch.float32
            es = 16 if prec == "double" else 8
            pr = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=prec, transform=transform)
            pr.initFFT(dfft.GlobalSize(n, n, n), None, True, data=(m, m, m))
            ordp = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=prec, transform=transform)
            ordp.initFFT(dfft.GlobalSize(n, n, n), None, True)
            g = torch.Generator(device=dev).manual_seed(1)
            x = torch.randn((m, m, m), generator=g, dtype=rdt, device=dev)
            if not r2c:
                x = torch.complex(x, torch.randn((m, m, m), generator=g, dtype=rdt, device=dev))
            spec = torch.empty(tuple(pr.getOutSize()), dtype=cdt, device=dev)
            back = torch.empty_like(x)
            emb = torch.empty((n, n, n), dtype=x.dtype, device=dev)  # the caller's doubled-grid field
            full_back = torch.empty_like(emb)

            def pr_fwd():
                pr.execR2C(spec, x) if r2c else pr.execC2C(spec, x, dfft.FORWARD)

            def pr_inv():
                pr.execC2R(back, spec) if r2c else pr.execC2C(back, spec, dfft.INVERSE)

            def ord_fwd():
                emb.zero_()
                emb[:m, :m, :m] = x
                ordp.execR2C(spec, emb) if r2c else ordp.execC2C(spec, emb, dfft.FORWARD)

            def ord_inv():
                ordp.execC2R(full_back, spec) if r2c else ordp.execC2C(full_back, spec, dfft.INVERSE)
                back.copy_(full_back[:m, :m, :m])

            def window(fn):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / args.reps

            fns = {"pruned_fwd": pr_fwd, "ordinary_fwd": ord_fwd, "pruned_inv": pr_inv, "ordinary_inv": ord_inv}
            pr_fwd()  # the inverses take a spectrum
            for fn in fns.values():  # warm-up: modules, tables, torch's kernels
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            times = {name: [] for name in fns}
            for _ in range(args.windows):
                for name, fn in fns.items():
                    times[name].append(window(fn))
            # whether the pruned spectrum equals the embedded one bit for bit, and the inverses' blocks
            pr_fwd()
            s_pr = spec.clone()
            ord_fwd()
            same_fwd = bool(torch.equal(s_pr, spec))
            pr_inv()
            b_pr = back.clone()
            ord_inv()
            same_inv = bool(torch.equal(b_pr, back))
            steps = {}
            pr.enableTimer(True)
            for name, fn in (("fwd", pr_fwd), ("inv", pr_inv)):
                fn()
                torch.cuda.synchronize()
                steps[name] = [(label, round(ms, 4)) for label, ms in pr.stepTimes()]
            pr.enableTimer(False)
            fl = floors(n, m, es, r2c)
            med = {name: sorted(v)[len(v) // 2] for name, v in times.items()}
            res = {"card": info, "n": n, "m": m, "precision": prec, "transform": transform, "ms_median": {a: round(b, 4) for a, b in med.items()},
                   "ms_windows": {a: [round(t, 4) for t in b] for a, b in times.items()}, "pruned_steps_ms": steps,
                   "floor_ms": {a: round(b / HBM_BYTES_PER_S * 1e3, 4) for a, b in fl.items()},
                   "speedup_fwd": round(med["ordinary_fwd"] / med["pruned_fwd"], 3), "speedup_inv": round(med["ordinary_inv"] / med["pruned_inv"], 3),
                   "work_bytes": {"pruned": pr.getWorkSizeDevice(), "ordinary": ordp.getWorkSizeDevice()},
                   "physical_bytes": {"pruned": x.numel() * x.element_size(), "ordinary": emb.numel() * emb.element_size()},
                   "forward_bit_identical": same_fwd, "inverse_bit_identical": same_inv}
            print(json.dumps(res), flush=True)
            results.append(res)
            pr.destroy()
            ordp.destroy()
            del x, spec, back, emb, full_back
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
