"""16-bit plans (DFFT_F16 / DFFT_BF16) against the f32 plan of the same geometry on one GPU.

A 512^3 grid, C2C and R2C / C2R, forward and inverse.  For each it times
  * the one-rank slab plan in FP16, BF16 and f32, in alternating windows of CUDA-event-timed execs (the whole exec);
  * each pass from the step timer (median over --steps timed execs), its bytes (every pass reads and writes its arrays
    once: 2 x elements x 4 bytes for a 16-bit C2C pass, R2C / C2R: 2-byte reals on the real side) and the rate and share of
    3.35 TB/s (the H100 SXM data sheet) they give;
  * the f32 plan's sequential schedule as well: the one-rank f32 slab C2C forward runs the fused z + y stage, so the same
    transform also runs as a 1 x 1 pencil plan (sequential z, y, x passes), in both precisions;
  * the rel-L2 error of the 16-bit forward against the float64 transform of the widened input, and of the round trip with
    (1, 1/N).
The card's name, power limit and max SM clock are read in the same run.  A report, not a gate: one JSON line per case
(and all of them to --out).

    python tools/half_bench.py [--n 512] [--reps 10] [--windows 5] [--steps 5] [--out half_bench.json]
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
PRECS = ("half", "bfloat16", "float")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def pass_bytes(label, n, es, r2c):
    """bytes a pass must move: one read and one write of its arrays (the z pass of R2C / C2R: reals on one side); the fused
    z + y stage counts as its two passes"""
    nzc = n // 2 + 1 if r2c else n
    grid = n * n * nzc * es
    if label.startswith("zy") or label.startswith("yz"):
        return 2 * 2 * grid
    if label.startswith("z") and r2c:
        return n * n * n * es // 2 + grid
    return 2 * grid


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10, help="execs per timed window")
    ap.add_argument("--windows", type=int, default=5, help="alternating windows per plan")
    ap.add_argument("--steps", type=int, default=5, help="step-timed execs per plan")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import distributedfft_b200 as dfft

    if not torch.cuda.is_available():
        raise SystemExit("half_bench.py needs a CUDA device")
    n = args.n
    N = n ** 3
    info = card()
    comm = dfft.Comm(0, 1, None, 0)
    results = []
    for transform in ("c2c", "r2c"):
        r2c = transform == "r2c"
        nzc = n // 2 + 1 if r2c else n
        kinds = [("slab", p) for p in PRECS] + ([("pencil", "half"), ("pencil", "float")] if not r2c else [])
        plans, bufs = {}, {}
        g = torch.Generator(device="cuda").manual_seed(1)
        x64 = torch.randn((n, n, n) + (() if r2c else (2,)), generator=g, device="cuda") * 0.25
        for decomp, prec in kinds:
            cls = dfft.MPIcuFFT_Slab if decomp == "slab" else dfft.MPIcuFFT_Pencil
            pl = cls(dfft.Configurations(), comm, precision=prec, transform=transform)
            pl.initFFT(dfft.GlobalSize(n, n, n), None if decomp == "slab" else dfft.Pencil_Partition(1, 1), True)
            dt = {"half": torch.float16, "bfloat16": torch.bfloat16, "float": torch.float32}[prec]
            x = x64.to(dt)
            spec = torch.empty((n, n, nzc, 2), dtype=dt, device="cuda")
            back = torch.empty_like(x)
            plans[(decomp, prec)] = pl
            bufs[(decomp, prec)] = (x, spec, back)

        def run(key, inverse):
            pl, (x, spec, back) = plans[key], bufs[key]
            if inverse:
                pl.execC2R(back, spec) if r2c else pl.execC2C(back, spec, dfft.INVERSE)
            else:
                pl.execR2C(spec, x) if r2c else pl.execC2C(spec, x, dfft.FORWARD)

        def window(key, inverse):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                run(key, inverse)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / args.reps

        for key in plans:  # warm-up: modules, tables; the inverses take a spectrum
            for inverse in (0, 1):
                for _ in range(3):
                    run(key, inverse)
        torch.cuda.synchronize()
        for inverse in (0, 1):
            times = {key: [] for key in plans}
            for _ in range(args.windows):
                for key in plans:
                    times[key].append(window(key, inverse))
            steps = {}
            for key, pl in plans.items():
                pl.enableTimer(True)
                per = {}
                for _ in range(args.steps):
                    run(key, inverse)
                    torch.cuda.synchronize()
                    for label, ms in pl.stepTimes():
                        per.setdefault(label, []).append(ms)
                pl.enableTimer(False)
                es = 8 if key[1] == "float" else 4
                rows = []
                for label, v in per.items():
                    ms = sorted(v)[len(v) // 2]
                    b = pass_bytes(label, n, es, r2c) if "pass" in label and "tail" not in label else 0
                    rows.append({"label": label, "ms": round(ms, 4), "bytes": b,
                                 "TB/s": round(b / ms / 1e9, 3) if b and ms > 0 else None,
                                 "share_of_3.35": round(b / ms / 1e9 / 3.35, 3) if b and ms > 0 else None})
                steps[f"{key[0]}/{key[1]}"] = rows
            med = {f"{k[0]}/{k[1]}": round(sorted(v)[len(v) // 2], 4) for k, v in times.items()}
            res = {"card": info, "n": n, "transform": transform, "direction": "inverse" if inverse else "forward", "exec_ms_median": med,
                   "exec_ms_windows": {f"{k[0]}/{k[1]}": [round(t, 4) for t in v] for k, v in times.items()},
                   "steps": steps}
            print(json.dumps(res), flush=True)
            results.append(res)
        # errors against float64: forward unscaled, round trip with (1, 1/N)
        xd = x64.double() if r2c else torch.view_as_complex(x64.double())
        for prec in ("half", "bfloat16"):
            pl, (x, spec, back) = plans[("slab", prec)], bufs[("slab", prec)]
            pl.setScale(1.0, 1.0 / N)
            run(("slab", prec), 0)
            run(("slab", prec), 1)
            torch.cuda.synchronize()
            xw = x.double() if r2c else torch.view_as_complex(x.double())
            ref = torch.fft.rfftn(xw) if r2c else torch.fft.fftn(xw)
            e_fwd = float(torch.linalg.vector_norm(torch.view_as_complex(spec.double()) - ref) / torch.linalg.vector_norm(ref))
            del ref
            bk = back.double() if r2c else torch.view_as_complex(back.double())
            e_rt = float(torch.linalg.vector_norm(bk - xw) / torch.linalg.vector_norm(xw))
            e_in = float(torch.linalg.vector_norm(xw - xd) / torch.linalg.vector_norm(xd))
            res = {"card": info, "n": n, "transform": transform, "precision": prec, "forward_rel_l2": e_fwd, "round_trip_rel_l2": e_rt,
                   "input_rounding_rel_l2": e_in}
            print(json.dumps(res), flush=True)
            results.append(res)
        for pl in plans.values():
            pl.destroy()
        del plans, bufs, x64, xd
        torch.cuda.empty_cache()
    comm.destroy()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
