"""Spectral weights (dfft_plan_set_weights) against what a caller does without them, on one GPU.

A 512^3 grid: C2C f64, R2C / C2R f64 and f32, forward and inverse.  For each it times, in alternating windows of
CUDA-event-timed execs:
  (a) the unweighted exec of the one-rank slab plan;
  (b) the weighted exec, all three axes weighted;
  (c) the unweighted exec and one torch multiply by the broadcast W (forward: of the output; inverse: of a copy of the
      input, which the exec then transforms), what a caller does today;
  (d) the weighted plan with every pointer NULL: the sequential schedule with the unweighted kernels.  For the one-rank
      512^3 C2C plan, (a) runs the fused z + y stage and (b) the sequential schedule, so (d) - (a) is the schedule's cost
      and (b) - (d) the multiply's;
  (e) C2C f64 only: (d) with DFFT_TMA=0, the sequential schedule with the register-fed x pass the weighted plan runs
      (its 1024-point and longer TILED passes have no TMA-fed twin).
It also checks that (b) and (c) agree.  The card's name, power limit and max SM clock are read in the same run.  A report,
not a gate: one JSON line per case (and all of them to --out).

    python tools/weights_bench.py [--n 512] [--reps 10] [--windows 5] [--out weights_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--reps", type=int, default=10, help="execs per timed window")
    ap.add_argument("--windows", type=int, default=5, help="alternating windows per variant")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import distributedfft_b200 as dfft

    if not torch.cuda.is_available():
        sys.exit("weights_bench.py needs a GPU")
    torch.cuda.set_device(0)
    n = args.n
    info = card()
    print(json.dumps({"card": info}), flush=True)
    results = []
    for transform, prec in (("c2c", "double"), ("r2c", "double"), ("r2c", "float")):
        c2c = transform == "c2c"
        rdt = torch.float64 if prec == "double" else torch.float32
        cdt = torch.complex128 if prec == "double" else torch.complex64
        nzc = n if c2c else n // 2 + 1

        def make(weights):
            p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=prec, transform=transform)
            p.initFFT(dfft.GlobalSize(n, n, n), None, True)
            if weights is not None:
                p.setWeights(*weights)
            return p

        g = torch.Generator(device="cuda").manual_seed(1)
        ws = [torch.complex(torch.rand(k, generator=g, device="cuda", dtype=rdt), torch.rand(k, generator=g, device="cuda", dtype=rdt))
              for k in (n, n, nzc)]
        W = ws[0][:, None, None] * ws[1][None, :, None] * ws[2][None, None, :]
        plain, wplan, nplan = make(None), make(ws), make([None, None, None])
        phys = torch.rand((n, n, n), generator=g, device="cuda", dtype=rdt)
        if c2c:
            phys = torch.complex(phys, torch.rand((n, n, n), generator=g, device="cuda", dtype=rdt))
        spec = torch.empty((n, n, nzc), dtype=cdt, device="cuda")
        tmp = torch.empty_like(spec)
        out_phys = torch.empty_like(phys)

        def run(plan, inverse):
            if c2c:
                plan.execC2C(out_phys if inverse else spec, tmp if inverse else phys, dfft.INVERSE if inverse else dfft.FORWARD)
            elif inverse:
                plan.execC2R(out_phys, tmp)
            else:
                plan.execR2C(spec, phys)

        plain.execR2C(spec, phys) if not c2c else plain.execC2C(spec, phys, dfft.FORWARD)
        src = spec.clone()
        for inverse in (0, 1):
            def a():
                if inverse:
                    tmp.copy_(src)
                run(plain, inverse)

            def b():
                if inverse:
                    tmp.copy_(src)
                run(wplan, inverse)

            def c():
                if inverse:
                    torch.mul(src, W, out=tmp)
                    run(plain, inverse)
                else:
                    run(plain, inverse)
                    spec.mul_(W)

            def d():
                if inverse:
                    tmp.copy_(src)
                run(nplan, inverse)

            def e():
                os.environ["DFFT_TMA"] = "0"
                try:
                    d()
                finally:
                    del os.environ["DFFT_TMA"]

            variants = {"a_unweighted": a, "b_weighted": b, "c_unweighted_plus_torch_multiply": c, "d_sequential_unweighted": d}
            if c2c and prec == "double":
                variants["e_sequential_register_fed"] = e
            # the copy of the inverse input is part of (a), (b) and (d) so that each reads a fresh spectrum, as (c) does
            copy_ms = 0.0
            if inverse:
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                for _ in range(3):
                    tmp.copy_(src)
                ev0.record()
                for _ in range(args.reps):
                    tmp.copy_(src)
                ev1.record()
                torch.cuda.synchronize()
                copy_ms = ev0.elapsed_time(ev1) / args.reps
            times = {k: [] for k in variants}
            for fn in variants.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            for _ in range(args.windows):
                for name, fn in variants.items():
                    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    ev0.record()
                    for _ in range(args.reps):
                        fn()
                    ev1.record()
                    torch.cuda.synchronize()
                    times[name].append(ev0.elapsed_time(ev1) / args.reps)
            # (b) against (c): the same values up to rounding
            b()
            got = (out_phys if inverse else spec).clone()
            c()
            want = out_phys if inverse else spec
            err = float(torch.linalg.vector_norm(got - want) / torch.linalg.vector_norm(want))
            med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
            row = {"transform": transform, "precision": prec, "n": n, "direction": "inverse" if inverse else "forward", "card": info,
                   "median_ms": {k: round(v, 4) for k, v in med.items()}, "min_ms": {k: round(min(v), 4) for k, v in times.items()},
                   "input_copy_ms": round(copy_ms, 4), "b_over_c": round(med["b_weighted"] / med["c_unweighted_plus_torch_multiply"], 3),
                   "rel_l2_b_vs_c": err}
            print(json.dumps(row), flush=True)
            results.append(row)
        for p in (plain, wplan, nplan):
            p.destroy()
        del W, phys, spec, tmp, out_phys
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
