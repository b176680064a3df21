"""DCT-I plans on one GPU (one-rank slab) against the DCT-II plan of nearly the same bytes and against the even-extension
route a caller without type-I kinds takes.

    python tools/r2r1_bench.py [--steps 10] [--rounds 3] [--n 512] [--precs f64,f32]

Cases, for each precision:
  - pass bandwidth: the (dct1, dct1, dct1) plan of (n+1)^3 against the DFFT_DCT plan of n^3, forward, per pass from the
    step timer; a pass reads and writes every real once (2 * sizeof(T) bytes per point), against the data-sheet 3.35 TB/s
    of an H100 SXM;
  - whole transform, cubic: the (n+1)^3 DCT-I plan against torch building the (2n)^3 even extension, the R2HC plan of (2n)^3
    and torch copying out the [0, n]^3 block of real parts (for k <= n the halfcomplex line holds Re X_k, which is y_k);
  - whole transform, Chebyshev channel: (dct1, r2hc, r2hc) on (n+1) x n x n against the same route along x only.
Windows of `steps` execs alternate between the routes on one stream, `rounds` times, timed with CUDA events (best window
reported).  Prints one JSON line per precision with the GPU's name, power limit and maximum SM clock read in the same run.
Nothing is gated on the numbers.
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


def plan(transform, shape, pname):
    p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=pname, transform=transform)
    p.initFFT(dfft.GlobalSize(*shape), None, True)
    return p


def timed(fn, steps, rounds):
    fn()
    torch.cuda.synchronize()
    best = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        best.append(round(e0.elapsed_time(e1) / steps, 4))
    return best


def step_times(p, out, x):
    p.execR2R(out, x, dfft.FORWARD)  # the first exec loads the kernels
    torch.cuda.synchronize()
    p.enableTimer(True)
    p.execR2R(out, x, dfft.FORWARD)
    p.wait()
    st = [(lbl, round(v, 5)) for lbl, v in p.stepTimes()]
    p.enableTimer(False)
    return st


def even_ext(x, axes):
    """the 2n-point even extension x_0 .. x_n, x_{n-1} .. x_1 along each of `axes`"""
    for a in axes:
        n = x.shape[a] - 1
        x = torch.cat([x, x.narrow(a, 1, n - 1).flip(a)], dim=a)
    return x.contiguous()


def run(n, prec, steps, rounds, gpu):
    pname = "double" if prec == "f64" else "float"
    rdt = torch.float64 if prec == "f64" else torch.float32
    es = 8 if prec == "f64" else 4
    g = torch.Generator(device="cuda").manual_seed(1)
    res = {"n": n, "prec": prec, "steps": steps, "gpu": gpu, "peak_tb_per_s": PEAK_TBS}

    # pass bandwidth: type-I passes on (n+1)^3 against the DCT-II passes on n^3
    for name, transform, m in (("dct1", ("dct1",) * 3, n + 1), ("dct2", "dct", n)):
        x = torch.rand((m,) * 3, generator=g, device="cuda", dtype=rdt)
        y = torch.empty_like(x)
        p = plan(transform, (m,) * 3, pname)
        st = step_times(p, y, x)
        res[f"{name}_step_ms"] = st
        res[f"{name}_pass_tb_per_s"] = [round(m ** 3 * 2 * es / (v * 1e-3) / 1e12, 3) for _, v in st if v > 0]
        res[f"{name}_exec_ms"] = timed(lambda: p.execR2R(y, x, dfft.FORWARD), steps, rounds)
        p.destroy()
        del x, y
        torch.cuda.empty_cache()

    # whole transforms against the even-extension route
    for case, names, shape, ext_axes in (("cube", ("dct1",) * 3, (n + 1,) * 3, (0, 1, 2)),
                                         ("channel", ("dct1", "r2hc", "r2hc"), (n + 1, n, n), (0,))):
        x = torch.rand(shape, generator=g, device="cuda", dtype=rdt)
        y = torch.empty_like(x)
        p = plan(names, shape, pname)
        eshape = tuple(2 * (s - 1) if a in ext_axes else s for a, s in enumerate(shape))
        q = plan(("r2hc",) * 3, eshape, pname)
        ebuf = torch.empty(eshape, device="cuda", dtype=rdt)
        eout = torch.empty_like(ebuf)
        yw = torch.empty_like(x)

        def route():
            ebuf.copy_(even_ext(x, ext_axes))
            q.execR2R(eout, ebuf, dfft.FORWARD)
            yw.copy_(eout[:shape[0], :shape[1], :shape[2]])

        p.execR2R(y, x, dfft.FORWARD)
        route()
        torch.cuda.synchronize()
        diff = float(torch.linalg.norm(y - yw) / torch.linalg.norm(yw))
        a, b = [], []
        for _ in range(rounds):
            a += timed(lambda: p.execR2R(y, x, dfft.FORWARD), steps, 1)
            b += timed(route, steps, 1)
        res[case] = {"shape": list(shape), "type1_ms": a, "route_ms": b, "route_over_type1": round(min(b) / min(a), 3), "rel_diff": diff}
        p.destroy(); q.destroy()
        del x, y, ebuf, eout, yw
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
        sys.exit("r2r1_bench.py needs a GPU")
    gpu = gpu_identity()
    for prec in args.precs.split(","):
        run(args.n, prec, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
