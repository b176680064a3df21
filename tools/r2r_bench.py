"""DCT plans against C2C and R2C plans of the same grid on one GPU (one-rank slab).

    python tools/r2r_bench.py [--steps 20] [--rounds 3] [--shapes 256,512] [--precs f64,f32]

For each grid and precision the DCT, C2C and R2C plans exist side by side; windows of `steps` forward execs and of `steps`
inverse execs alternate between them on one stream, `rounds` times, timed with CUDA events (best window reported).  One
timed exec per plan and direction gives the per-pass step times; the effective bandwidth of a pass counts one read and one
write of every element (2 * sizeof(T) bytes per point for DCT / DST, 2 * 2 * sizeof(T) for C2C) against the data-sheet
3.35 TB/s of an H100 SXM.  Prints one JSON line per grid and precision, with the GPU's name, power limit and maximum SM
clock read in the same run.
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
    shape = (n, n, n)
    pts = n ** 3
    rdt = torch.float64 if prec == "f64" else torch.float32
    cdt = torch.complex128 if prec == "f64" else torch.complex64
    es = 8 if prec == "f64" else 4
    g = torch.Generator(device="cuda").manual_seed(1)
    plans, bufs = {}, {}
    for t in ("dct", "c2c", "r2c"):
        p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if prec == "f64" else "float", transform=t)
        p.initFFT(dfft.GlobalSize(*shape), None, True)
        plans[t] = p
    x = torch.rand(shape, generator=g, device="cuda", dtype=rdt)
    bufs["dct"] = (x, torch.empty_like(x))
    xc = torch.complex(x, torch.rand(shape, generator=g, device="cuda", dtype=rdt))
    bufs["c2c"] = (xc, torch.empty_like(xc))
    bufs["r2c"] = (x, torch.empty((n, n, n // 2 + 1), device="cuda", dtype=cdt))
    stream = torch.cuda.current_stream()

    def ex(t, inverse):
        p, (a, b) = plans[t], bufs[t]
        if t == "dct":
            p.execR2R(a if inverse else b, b if inverse else a, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)
        elif t == "c2c":
            p.execC2C(a if inverse else b, b if inverse else a, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)
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
    bw = {}
    for key, lst in steps_ms.items():
        if key.startswith("r2c"):
            continue
        per_pt = 2 * es * (2 if key.startswith("c2c") else 1)
        bw[key] = [round(pts * per_pt / (v * 1e-3) / 1e12, 3) for _, v in lst if v > 0]
    print(json.dumps({"shape": list(shape), "prec": prec, "steps": steps, "ms": ms, "best_ms": best,
                      "dct_fwd_over_c2c_fwd": round(best["dct_fwd"] / best["c2c_fwd"], 4),
                      "dct_inv_over_c2c_inv": round(best["dct_inv"] / best["c2c_inv"], 4), "step_ms": steps_ms,
                      "pass_tb_per_s": bw, "peak_tb_per_s": PEAK_TBS, "gpu": gpu}), flush=True)
    for p in plans.values():
        p.destroy()
    del x, xc, bufs
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--shapes", default="256,512")
    ap.add_argument("--precs", default="f64,f32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("r2r_bench.py needs a GPU")
    gpu = gpu_identity()
    for n in (int(s) for s in args.shapes.split(",")):
        for prec in args.precs.split(","):
            run(n, prec, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
