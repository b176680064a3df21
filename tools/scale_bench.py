"""Cost of the output scale (dfft_plan_set_scale) on one GPU: a scaled exec against an unscaled exec, and against an
unscaled exec followed by a separate `out.mul_(s)`, eager and replayed from a CUDA graph.

    python tools/scale_bench.py [--steps 20] [--rounds 3] [--cases all|name,name]

Cases: 512^3 complex-double forward and inverse, 256^3 complex-double forward, 1024^3 R2C f64 inverse (C2R), 64 fields of
64^3 complex-double (one launch).  Per case the four variants run in alternating windows of `steps` execs on one stream
(scaled, unscaled, unscaled + mul_, graph of unscaled + mul_), `rounds` times, timed with CUDA events.  The scaled output
must equal the unscaled output times s bit for bit.  Prints one JSON line per case with the ms per exec of every window
and the GPU's name, power limit and maximum SM clock, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402

CASES = {
    # name: (shape, transform, inverse, batch)
    "c2c_512_fwd": ((512, 512, 512), "c2c", 0, 1),
    "c2c_512_inv": ((512, 512, 512), "c2c", 1, 1),
    "c2c_256_fwd": ((256, 256, 256), "c2c", 0, 1),
    "c2r_1024_inv": ((1024, 1024, 1024), "r2c", 1, 1),
    "c2c_64x64_fwd": ((64, 64, 64), "c2c", 0, 64),
}


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def run_case(name, steps, rounds, gpu):
    shape, transform, inverse, batch = CASES[name]
    c2c = transform == "c2c"
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), None, True, batch=batch)
    nx, ny, nz = shape
    nzc = nz if c2c else nz // 2 + 1
    s = 1.0 / (nx * ny * nz)
    g = torch.Generator(device="cuda").manual_seed(1)
    spec_shape, real_shape = (batch, nx, ny, nzc), (batch, nx, ny, nz)
    if inverse:
        x = torch.complex(torch.rand(spec_shape, generator=g, device="cuda", dtype=torch.float64),
                          torch.rand(spec_shape, generator=g, device="cuda", dtype=torch.float64))
        if not c2c:  # a valid half spectrum: the forward transform of real data
            r = torch.rand(real_shape, generator=g, device="cuda", dtype=torch.float64)
            plan.execR2C(x, r)
            del r
        out = torch.empty(real_shape, device="cuda", dtype=torch.complex128 if c2c else torch.float64)
    else:
        x = torch.complex(torch.rand(real_shape, generator=g, device="cuda", dtype=torch.float64),
                          torch.rand(real_shape, generator=g, device="cuda", dtype=torch.float64))
        out = torch.empty(spec_shape, device="cuda", dtype=torch.complex128)
    stream = torch.cuda.current_stream()

    def exec_(st=stream):
        if c2c:
            plan.execC2C(out, x, dfft.INVERSE if inverse else dfft.FORWARD, stream=st)
        elif inverse:
            plan.execC2R(out, x, stream=st)
        else:
            plan.execR2C(out, x, stream=st)

    def set_scale(v):
        plan.setScale(*((1.0, v) if inverse else (v, 1.0)))

    real_view = (lambda t: torch.view_as_real(t)) if out.is_complex() else (lambda t: t)
    # bit identity: scaled == unscaled * s in float64
    set_scale(1.0)
    exec_()
    torch.cuda.synchronize()
    want = real_view(out) * s
    set_scale(s)
    exec_()
    torch.cuda.synchronize()
    identical = bool(torch.equal(real_view(out).view(torch.int64), want.view(torch.int64)))
    del want
    # graph of the unscaled exec followed by the separate multiply
    set_scale(1.0)
    exec_()
    torch.cuda.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        exec_(torch.cuda.current_stream())
        out.mul_(s)
    gr.replay()
    torch.cuda.synchronize()

    def window(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1) / steps, 5)

    def scaled():
        exec_()

    def unscaled_mul():
        exec_()
        out.mul_(s)

    res = {"scaled": [], "unscaled": [], "unscaled_then_mul": [], "graph_unscaled_then_mul": []}
    for _ in range(rounds):
        set_scale(s)
        exec_()  # setScale requires an eager exec; it is also the warm-up of the window
        res["scaled"].append(window(scaled))
        set_scale(1.0)
        exec_()
        res["unscaled"].append(window(exec_))
        res["unscaled_then_mul"].append(window(unscaled_mul))
        res["graph_unscaled_then_mul"].append(window(gr.replay))
    plan.wait()
    best = {k: min(v) for k, v in res.items()}
    print(json.dumps({"case": name, "shape": list(shape), "batch": batch, "transform": transform, "inverse": inverse, "scale": s,
                      "steps": steps, "ms_per_exec": res, "best_ms": best,
                      "scaled_over_unscaled": round(best["scaled"] / best["unscaled"], 4),
                      "saving_vs_mul_ms": round(best["unscaled_then_mul"] - best["scaled"], 5),
                      "saving_vs_graph_mul_ms": round(best["graph_unscaled_then_mul"] - best["scaled"], 5),
                      "scaled_equals_unscaled_times_s": identical, "gpu": gpu}), flush=True)
    del gr
    plan.destroy()
    del x, out
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cases", default="all")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("scale_bench.py needs a GPU")
    names = list(CASES) if args.cases == "all" else args.cases.split(",")
    gpu = gpu_identity()
    for name in names:
        run_case(name, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
