"""Interleaved multi-component plans against the permute route on one GPU.

For each workload ([X, Y, Z, C] complex fields, forward and inverse) it times
  (a) the interleaved plan (dfft_plan_create_interleaved) on the [X, Y, Z, C] tensor;
  (b) torch permute to [C, X, Y, Z], the batched plan (batch = C), permute back;
  (c) the batched plan on data already in [C, X, Y, Z] (reference);
in alternating windows of CUDA-event-timed execs on one stream (best and all windows), then the z pass of (a) and of (c)
from the per-step timer of a partial d = 1 exec (the full exec of (c) fuses z with y at 256^3 and 512^3), with its share of
the 3.35 TB/s HBM bound of the H100 SXM data sheet (one read and one write of the array: real side 8 bytes, complex side
16 bytes per value).  The card's name, power limit and maximum SM clock are read in the same run.  A report, not a gate: one JSON
line per case.

    python tools/components_bench.py [--reps 10] [--windows 5] [--precision double|float] [--transform c2c|r2c] [--out components_bench.json]
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
WORKLOADS = [((512, 512, 512), 3, "c2c"), ((256, 256, 256), 3, "c2c"), ((256, 256, 256), 3, "r2c"), ((64, 64, 64), 8, "c2c")]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--reps", type=int, default=10, help="execs per timed window")
    ap.add_argument("--windows", type=int, default=5, help="alternating windows per variant")
    ap.add_argument("--precision", choices=["double", "float"], default="double")
    ap.add_argument("--transform", choices=["c2c", "r2c"], default=None, help="only the workloads of this transform")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import distributedfft_b200 as dfft

    if not torch.cuda.is_available():
        sys.exit("components_bench needs a GPU")
    gpu = card()
    lines = []
    f64 = args.precision == "double"
    cdt, rdt = (torch.complex128, torch.float64) if f64 else (torch.complex64, torch.float32)
    for shape, comps, transform in WORKLOADS:
        if args.transform and transform != args.transform:
            continue

        def plan(c, b):
            p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=args.precision, transform=transform)
            p.initFFT(dfft.GlobalSize(*shape), None, True, batch=b, components=c)
            return p

        c2c = transform == "c2c"
        ilv, bat = plan(comps, 1), plan(1, comps)
        spec = shape if c2c else shape[:2] + (shape[2] // 2 + 1,)
        xr = torch.randn(shape + (comps,), dtype=cdt if c2c else rdt, device="cuda")
        # inverse input: a spectrum of real fields for C2R (X[0] and X[Nz/2] real along z)
        Xs = torch.randn(spec + (comps,), dtype=cdt, device="cuda") if c2c else torch.fft.rfftn(xr, dim=(0, 1, 2)).contiguous()
        s = torch.cuda.current_stream()

        def run(p, out, inp, direction, d=3, stream=s):
            if c2c:
                p.execC2C(out, inp, direction, d, stream=stream) if stream is not None else p.execC2C(out, inp, direction, d)
            elif direction == dfft.FORWARD:
                p.execR2C(out, inp, d, stream=stream) if stream is not None else p.execR2C(out, inp, d)
            else:
                p.execC2R(out, inp, d, stream=stream) if stream is not None else p.execC2R(out, inp, d)

        for direction, name in ((dfft.FORWARD, "forward"), (dfft.INVERSE, "inverse")):
            x = xr if direction == dfft.FORWARD else Xs
            ya = torch.empty((spec if direction == dfft.FORWARD else shape) + (comps,), dtype=Xs.dtype if direction == dfft.FORWARD else xr.dtype,
                             device="cuda")
            xc = x.permute(3, 0, 1, 2).contiguous()
            yc = ya.permute(3, 0, 1, 2).contiguous()

            def a():
                run(ilv, ya, x, direction)

            def b():
                t = x.permute(3, 0, 1, 2).contiguous()
                run(bat, yc, t, direction)
                ya.copy_(yc.permute(1, 2, 3, 0))

            def c():
                run(bat, yc, xc, direction)

            variants = {"a_interleaved": a, "b_permute_batched": b, "c_batched_planar": c}
            for f in variants.values():  # warm-up: module load, tables, kernel attributes
                f(); f()
            torch.cuda.synchronize()
            times = {k: [] for k in variants}
            for _ in range(args.windows):
                for k, f in variants.items():
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        f()
                    e1.record()
                    torch.cuda.synchronize()
                    times[k].append(e0.elapsed_time(e1) / args.reps)
            # z pass of (a) and (c): partial d = 1 execs (the z pass alone), timed by the step timer; one read and one write
            # of all C components
            steps = {}
            zin = xr if direction == dfft.FORWARD else Xs
            zout = torch.empty((spec if direction == dfft.FORWARD else shape) + (comps,), dtype=ya.dtype, device="cuda")
            nbytes = zin.numel() * zin.element_size() + zout.numel() * zout.element_size()
            zin_c, zout_c = zin.permute(3, 0, 1, 2).contiguous(), zout.permute(3, 0, 1, 2).contiguous()
            for k, p, o, i in (("a_interleaved", ilv, zout, zin), ("c_batched_planar", bat, zout_c, zin_c)):
                p.enableTimer(True)
                best = None
                for _ in range(5):
                    run(p, o, i, direction, 1, None)
                    zs = [ms for lbl, ms in p.stepTimes() if lbl.startswith("z pass")]
                    best = sum(zs) if best is None else min(best, sum(zs))
                p.enableTimer(False)
                z_ms = best
                steps[k] = {"z_pass_ms": round(z_ms, 4), "z_pass_hbm_fraction": round(nbytes / (z_ms * 1e-3) / HBM_BYTES_PER_S, 3) if z_ms else None}
            a()
            c()
            torch.cuda.synchronize()
            ok = bool(torch.equal(ya.permute(3, 0, 1, 2), yc)) if c2c else float((ya.permute(3, 0, 1, 2) - yc).abs().max() / yc.abs().max())
            line = {"gpu": gpu, "precision": args.precision, "shape": list(shape), "components": comps, "transform": transform, "direction": name,
                    "best_ms": {k: round(min(v), 4) for k, v in times.items()}, "all_ms": {k: [round(t, 4) for t in v] for k, v in times.items()},
                    "z_pass": steps, "a_vs_c": ok}
            print(json.dumps(line), flush=True)
            lines.append(line)
        ilv.destroy()
        bat.destroy()
        del x, xc, ya, yc, xr, Xs
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
