"""DCT-IV plans on one GPU (one-rank slab) against the DCT-II plan of the same bytes and against the route a caller without
type-IV kinds takes.

    python tools/r2r4_bench.py [--steps 10] [--rounds 3] [--n 512] [--precs f64,f32]

Cases, for each precision:
  - pass bandwidth: the (dct4, dct4, dct4) plan of n^3 against the DFFT_DCT plan of n^3, forward, per pass from the step
    timer; a pass reads and writes every real once (2 * sizeof(T) bytes per point), against the data-sheet 3.35 TB/s of an
    H100 SXM; and the whole execs of both plans in alternating windows;
  - whole transform, channel: (dct4, r2hc, r2hc) on n^3 against the same plan with x kept (dfft_plan_set_transform_axes)
    followed by a DCT-IV along x in torch: pre-twiddle exp(-i pi m / 2N), a 2N-point zero-padded complex FFT, post-twiddle
    exp(-i pi (2k + 1) / 4N) and twice the real part.
Windows of `steps` execs alternate between the routes on one stream, `rounds` times, timed with CUDA events (best window
reported).  Prints one JSON line per precision with the GPU's name, power limit and maximum SM clock read in the same run.
Nothing is gated on the numbers.
"""
import argparse
import json
import math
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


def plan(transform, shape, pname, transform_axes=None):
    p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=pname, transform=transform)
    p.initFFT(dfft.GlobalSize(*shape), None, True, transform_axes=transform_axes)
    return p


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return round(e0.elapsed_time(e1) / steps, 4)


def alternate(fa, fb, steps, rounds):
    fa(); fb()
    torch.cuda.synchronize()
    a, b = [], []
    for _ in range(rounds):
        a.append(timed(fa, steps))
        b.append(timed(fb, steps))
    return a, b


def step_times(p, out, x):
    p.execR2R(out, x, dfft.FORWARD)  # the first exec loads the kernels
    torch.cuda.synchronize()
    p.enableTimer(True)
    p.execR2R(out, x, dfft.FORWARD)
    p.wait()
    st = [(lbl, round(v, 5)) for lbl, v in p.stepTimes()]
    p.enableTimer(False)
    return st


def dct4_torch(x, cdt):
    """DCT-IV along dim 0 (scipy's dct(type=4)): y_k = 2 Re(exp(-i pi (2k+1) / 4N) sum_m x_m exp(-i pi m / 2N) W_2N^{mk})"""
    n = x.shape[0]
    m = torch.arange(n, device=x.device, dtype=x.dtype)
    pre = torch.exp(-1j * math.pi * m / (2 * n)).to(cdt).view(-1, 1, 1)
    post = torch.exp(-1j * math.pi * (2 * m + 1) / (4 * n)).to(cdt).view(-1, 1, 1)
    z = torch.fft.fft(x * pre, n=2 * n, dim=0)[:n]
    return 2 * (z * post).real


def run(n, prec, steps, rounds, gpu):
    pname = "double" if prec == "f64" else "float"
    rdt = torch.float64 if prec == "f64" else torch.float32
    cdt = torch.complex128 if prec == "f64" else torch.complex64
    es = 8 if prec == "f64" else 4
    g = torch.Generator(device="cuda").manual_seed(1)
    res = {"n": n, "prec": prec, "steps": steps, "gpu": gpu, "peak_tb_per_s": PEAK_TBS}

    # pass bandwidth: type-IV passes against the DCT-II passes on the same n^3 reals
    shape = (n,) * 3
    x = torch.rand(shape, generator=g, device="cuda", dtype=rdt)
    y4, y2 = torch.empty_like(x), torch.empty_like(x)
    p4, p2 = plan(("dct4",) * 3, shape, pname), plan("dct", shape, pname)
    for name, p, y in (("dct4", p4, y4), ("dct2", p2, y2)):
        st = step_times(p, y, x)
        res[f"{name}_step_ms"] = st
        res[f"{name}_pass_tb_per_s"] = [round(n ** 3 * 2 * es / (v * 1e-3) / 1e12, 3) for _, v in st if v > 0]
    a, b = alternate(lambda: p4.execR2R(y4, x, dfft.FORWARD), lambda: p2.execR2R(y2, x, dfft.FORWARD), steps, rounds)
    res["dct4_exec_ms"], res["dct2_exec_ms"] = a, b
    p4.destroy(); p2.destroy()

    # the channel against the kept-x plan plus a DCT-IV along x in torch
    names = ("dct4", "r2hc", "r2hc")
    p = plan(names, shape, pname)
    q = plan(names, shape, pname, transform_axes=(False, True, True))
    yq = torch.empty_like(x)
    yw = torch.empty_like(x)

    def route():
        q.execR2R(yq, x, dfft.FORWARD)
        yw.copy_(dct4_torch(yq, cdt))

    p.execR2R(y4, x, dfft.FORWARD)
    route()
    torch.cuda.synchronize()
    diff = float(torch.linalg.norm(y4 - yw) / torch.linalg.norm(yw))
    a, b = alternate(lambda: p.execR2R(y4, x, dfft.FORWARD), route, steps, rounds)
    res["channel"] = {"shape": list(shape), "type4_ms": a, "route_ms": b, "route_over_type4": round(min(b) / min(a), 3), "rel_diff": diff}
    p.destroy(); q.destroy()
    del x, y4, y2, yq, yw
    torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--precs", default="f64,f32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("r2r4_bench.py needs a GPU")
    gpu = gpu_identity()
    for prec in args.precs.split(","):
        run(args.n, prec, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
