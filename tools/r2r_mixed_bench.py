"""A mixed-boundary plan against the uniform DCT plan, the R2C plan of the same grid and the even-extension workaround on one
GPU (one-rank slab).

    python tools/r2r_mixed_bench.py [--steps 20] [--rounds 3] [--n 512] [--precs f64,f32]

Plans, side by side for each precision:
  - channel:  kinds (r2hc, r2hc, dct) on n^3 — periodic x and y, a Neumann wall along z;
  - dct:      the DFFT_DCT plan of n^3;
  - r2c:      the R2C plan of n^3;
  - r2c_ext:  the R2C plan of n x n x 2n, the even extension along z that a caller without per-axis kinds transforms
              instead (the copy kernel that builds the extension is not counted).
Windows of `steps` forward execs and of `steps` inverse execs alternate between the plans on one stream, `rounds` times,
timed with CUDA events (best window reported).  One timed exec per plan and direction gives the per-pass step times; the
effective bandwidth of a real-to-real pass counts one read and one write of every real (2 * sizeof(T) bytes per point)
against the data-sheet 3.35 TB/s of an H100 SXM.  Prints one JSON line per precision, with the GPU's name, power limit and
maximum SM clock read in the same run.  Nothing is gated on the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402

PEAK_TBS = 3.35


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def run(n, prec, steps, rounds, gpu):
    shape, ext = (n, n, n), (n, n, 2 * n)
    pts = n ** 3
    pname = "double" if prec == "f64" else "float"
    rdt = torch.float64 if prec == "f64" else torch.float32
    cdt = torch.complex128 if prec == "f64" else torch.complex64
    es = 8 if prec == "f64" else 4
    g = torch.Generator(device="cuda").manual_seed(1)
    specs = {"channel": (("r2hc", "r2hc", "dct"), shape), "dct": ("dct", shape), "r2c": ("r2c", shape), "r2c_ext": ("r2c", ext)}
    plans, bufs = {}, {}
    for t, (transform, s) in specs.items():
        p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=pname, transform=transform)
        p.initFFT(dfft.GlobalSize(*s), None, True)
        plans[t] = p
    x = torch.rand(shape, generator=g, device="cuda", dtype=rdt)
    bufs["channel"] = (x, torch.empty_like(x))
    bufs["dct"] = (x, torch.empty_like(x))
    bufs["r2c"] = (x, torch.empty((n, n, n // 2 + 1), device="cuda", dtype=cdt))
    xe = torch.cat([x, x.flip(2)], dim=2).contiguous()  # the even extension along z
    bufs["r2c_ext"] = (xe, torch.empty((n, n, n + 1), device="cuda", dtype=cdt))
    stream = torch.cuda.current_stream()

    def ex(t, inverse):
        p, (a, b) = plans[t], bufs[t]
        if t in ("channel", "dct"):
            p.execR2R(a if inverse else b, b if inverse else a, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)
        elif inverse:
            p.execC2R(a, b, stream=stream)
        else:
            p.execR2C(b, a, stream=stream)

    def window(t, inverse):
        ex(t, inverse)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            ex(t, inverse)
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    # the inverse input of each plan is its forward output
    for t in plans:
        ex(t, False)
    torch.cuda.synchronize()
    ms = {f"{t}_{d}": [] for t in plans for d in ("fwd", "inv")}
    for _ in range(rounds):
        for t in plans:
            for d, inv in (("fwd", False), ("inv", True)):
                ms[f"{t}_{d}"].append(round(window(t, inv), 5))
    steps_ms = {}
    for t, p in plans.items():
        p.enableTimer(True)
        for d, inv in (("fwd", False), ("inv", True)):
            ex(t, inv)
            p.wait()
            steps_ms[f"{t}_{d}"] = [(lbl, round(v, 5)) for lbl, v in p.stepTimes()]
        p.enableTimer(False)
    best = {k: min(v) for k, v in ms.items()}
    bw = {key: [round(pts * 2 * es / (v * 1e-3) / 1e12, 3) for _, v in lst if v > 0]
          for key, lst in steps_ms.items() if key.startswith(("channel", "dct"))}
    ratios = {f"channel_{d}_over_{t}_{d}": round(best[f"channel_{d}"] / best[f"{t}_{d}"], 4) for t in ("dct", "r2c", "r2c_ext") for d in ("fwd", "inv")}
    print(json.dumps({"shape": list(shape), "prec": prec, "steps": steps, "ms": ms, "best_ms": best, "ratios": ratios, "step_ms": steps_ms,
                      "pass_tb_per_s": bw, "peak_tb_per_s": PEAK_TBS, "gpu": gpu}), flush=True)
    for p in plans.values():
        p.destroy()
    del x, xe, bufs
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--precs", default="f64,f32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("r2r_mixed_bench.py needs a GPU")
    gpu = gpu_identity()
    for prec in args.precs.split(","):
        run(args.n, prec, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
