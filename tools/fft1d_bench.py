"""Times one-rank 1D plans (dfft_plan_create_1d) forward and inverse at N = 2^20 .. 2^30 against torch.fft.fft / ifft
(cuFFT) on the same GPU.

Each size warms up both, then runs `--rounds` rounds that alternate the plan and cuFFT, each round `--reps` execs between
two CUDA events; the median per exec is reported.  The GPU's name, power limit and maximum SM clock are read in the same
run.  Both transforms hold their buffers at once: in f64 2^30 points need more than 80 GB (in, out, the plan's two work
slots and cuFFT's output), so f64 runs end at 2^29 there.  python tools/fft1d_bench.py [--precision double|float] [--min 20] [--max 30] [--json out.json]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="double", choices=["double", "float"])
    ap.add_argument("--min", type=int, default=20)
    ap.add_argument("--max", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    import distributedfft_b200 as dfft
    if not torch.cuda.is_available():
        raise SystemExit("fft1d_bench needs a GPU")
    torch.cuda.set_device(0)
    cdt = torch.complex128 if a.precision == "double" else torch.complex64
    rows = []
    print(f"# {torch.cuda.get_device_name(0)} | {gpu_info()} | {a.precision}")
    print(f"{'N':>6} {'factors':>18} {'fwd ms':>9} {'cuFFT fwd':>10} {'inv ms':>9} {'cuFFT inv':>10}")
    for L in range(a.min, a.max + 1):
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
        times = {"fwd": [], "inv": [], "cufft_fwd": [], "cufft_inv": []}
        for fn in (fwd, inv, ref_f, ref_i):
            fn()
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            times["fwd"].append(timed(fwd, a.reps))
            times["cufft_fwd"].append(timed(ref_f, a.reps))
            times["inv"].append(timed(inv, a.reps))
            times["cufft_inv"].append(timed(ref_i, a.reps))
        med = {k: statistics.median(v) for k, v in times.items()}
        rows.append({"log2n": L, "factors": f, **med, "precision": a.precision})
        print(f"  2^{L:2d} {str(f):>18} {med['fwd']:9.3f} {med['cufft_fwd']:10.3f} {med['inv']:9.3f} {med['cufft_inv']:10.3f}", flush=True)
        plan.destroy()
        del x, y, xv
        torch.cuda.empty_cache()
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"gpu": torch.cuda.get_device_name(0), "info": gpu_info(), "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
