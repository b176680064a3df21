"""Times one-rank 1D plans (dfft_plan_create_1d) forward and inverse at N = 2^20 .. 2^30 against torch.fft.fft / ifft
(cuFFT) on the same GPU.  --natural adds the natural-order plan (dfft_plan_create_1d_natural) as a third arm of the same
rounds; --profile then also lists every kernel's time per exec of both 1D plans (torch.profiler, a run of its own after the
timed rounds), so that the transposing z pass stands next to the scrambled plan's z pass.

Each size warms up both, then runs `--rounds` rounds that alternate the plan and cuFFT, each round `--reps` execs between
two CUDA events; the median per exec is reported.  The GPU's name, power limit and maximum SM clock are read in the same
run.  Both transforms hold their buffers at once: in f64 2^30 points need more than 80 GB (in, out, the plan's two work
slots and cuFFT's output), so f64 runs end at 2^29 there.
python tools/fft1d_bench.py [--precision double|float] [--min 20] [--max 30 | --sizes 20,24,29] [--natural] [--profile]
                            [--json out.json]"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001 - the report still names the device below
        return f"nvidia-smi unavailable ({e})"


def timed(fn, reps):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def kernel_times(fn, execs=5):
    """{kernel name: device ms per exec} of fn under torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(execs):
            fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            out[ev.key] = t / 1000.0 / execs
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="double", choices=["double", "float"])
    ap.add_argument("--min", type=int, default=20)
    ap.add_argument("--max", type=int, default=30)
    ap.add_argument("--sizes", default=None, help="comma-separated log2 N to time instead of --min .. --max")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    ap.add_argument("--natural", action="store_true", help="also time the natural-order plan, alternating with the others")
    ap.add_argument("--profile", action="store_true", help="with --natural: kernel times per exec of both 1D plans")
    a = ap.parse_args()
    import torch

    import distributedfft_b200 as dfft
    if not torch.cuda.is_available():
        raise SystemExit("fft1d_bench needs a GPU")
    torch.cuda.set_device(0)
    cdt = torch.complex128 if a.precision == "double" else torch.complex64
    rows = []
    print(f"# {torch.cuda.get_device_name(0)} | {gpu_info()} | {a.precision}")
    print(f"{'N':>6} {'factors':>18} {'fwd ms':>9} {'cuFFT fwd':>10} {'inv ms':>9} {'cuFFT inv':>10}" +
          (f" {'nat fwd':>9} {'nat inv':>9}" if a.natural else ""))
    for L in [int(v) for v in a.sizes.split(",")] if a.sizes else range(a.min, a.max + 1):
        n = 1 << L
        plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(0, 1, None, 0), precision=a.precision, transform="c2c")
        plan.initFFT(None, signal=n)
        f = tuple(plan.getFactors())
        x = torch.randn(n, dtype=cdt, device="cuda")
        y = torch.empty(f, dtype=cdt, device="cuda")
        xv = x.view(f)
        fwd = lambda: plan.execC2C(y, xv, dfft.FORWARD, stream=torch.cuda.current_stream())  # noqa: E731
        inv = lambda: plan.execC2C(xv, y, dfft.INVERSE, stream=torch.cuda.current_stream())  # noqa: E731
        ref_f = lambda: torch.fft.fft(x)  # noqa: E731
        ref_i = lambda: torch.fft.ifft(x)  # noqa: E731
        arms = {"fwd": fwd, "cufft_fwd": ref_f, "inv": inv, "cufft_inv": ref_i}
        if a.natural:  # the natural-order plan of the same factors, its own output [N3][N2][N1]
            nat = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(0, 1, None, 0), precision=a.precision, transform="c2c")
            nat.initFFT(None, signal=n, factors=f, natural=True)
            yn = torch.empty(f[::-1], dtype=cdt, device="cuda")
            arms["nat_fwd"] = lambda: nat.execC2C(yn, xv, dfft.FORWARD, stream=torch.cuda.current_stream())  # noqa: E731
            arms["nat_inv"] = lambda: nat.execC2C(xv, yn, dfft.INVERSE, stream=torch.cuda.current_stream())  # noqa: E731
        times = {k: [] for k in arms}
        for fn in arms.values():
            fn()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, fn in arms.items():
                times[k].append(timed(fn, a.reps))
        med = {k: statistics.median(v) for k, v in times.items()}
        row = {"log2n": L, "factors": f, **med, "precision": a.precision}
        print(f"  2^{L:2d} {str(f):>18} {med['fwd']:9.3f} {med['cufft_fwd']:10.3f} {med['inv']:9.3f} {med['cufft_inv']:10.3f}" +
              (f" {med['nat_fwd']:9.3f} {med['nat_inv']:9.3f}" if a.natural else ""), flush=True)
        if a.natural and a.profile:
            row["kernels"] = {k: kernel_times(arms[k]) for k in ("fwd", "nat_fwd", "inv", "nat_inv")}
            for k, ks in row["kernels"].items():
                print(f"    {k}: " + "; ".join(f"{name[:120]} {ms:.3f} ms" for name, ms in sorted(ks.items(), key=lambda kv: -kv[1])), flush=True)
        rows.append(row)
        plan.destroy()
        if a.natural:
            nat.destroy()
            del yn
        del x, y, xv
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"gpu": torch.cuda.get_device_name(0), "info": gpu_info(), "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
