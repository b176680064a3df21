"""Eager execs against CUDA graph replays of the same exec, one GPU, one-rank slab C2C plans.

    python tools/graph_bench.py [--shapes 64,128,256,512] [--steps 20] [--warmup 5] [--prec f64|f32]

For each N^3: warm-up execs of both directions, then one forward and one inverse exec are captured into graphs
(torch.cuda.graph).  Eager execs and replays are timed with CUDA events on one stream, in alternating windows of `steps`
transforms (eager, graph, eager, graph), and each window's ms per transform is reported.  A replay's output must equal
the eager output bit for bit on the same input.  Prints one JSON line per shape, with the GPU's name, power limit and
maximum SM clock.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="64,128,256,512")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--prec", default="f64", choices=["f64", "f32"])
    args = ap.parse_args()
    f64 = args.prec == "f64"
    rdt, cdt = (torch.float64, torch.complex128) if f64 else (torch.float32, torch.complex64)
    gpu = gpu_identity()
    stream = torch.cuda.current_stream()
    for n in (int(v) for v in args.shapes.split(",")):
        plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform="c2c")
        plan.initFFT(dfft.GlobalSize(n, n, n), None, True)
        g = torch.Generator(device="cuda").manual_seed(1234)
        x = torch.complex(torch.rand(n ** 3, generator=g, device="cuda", dtype=rdt) * 255,
                          torch.rand(n ** 3, generator=g, device="cuda", dtype=rdt) * 255)
        out = torch.empty_like(x)
        back = torch.empty_like(x)
        fwd = lambda s: plan.execC2C(out, x, dfft.FORWARD, stream=s)  # noqa: E731
        inv = lambda s: plan.execC2C(back, out, dfft.INVERSE, stream=s)  # noqa: E731
        for _ in range(args.warmup):
            fwd(stream)
            inv(stream)
        plan.wait()
        graphs = {}
        for name, fn in (("forward", fwd), ("inverse", inv)):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                fn(torch.cuda.current_stream())
            gr.replay()  # the first launch uploads the graph
            graphs[name] = gr
        torch.cuda.synchronize()
        # same input, same kernels: bit-identical
        fwd(stream)
        ref = out.clone()
        out.zero_()
        graphs["forward"].replay()
        torch.cuda.synchronize()
        identical = bool(torch.equal(out, ref))

        def window(fn):
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                fn()
            e1.record(stream)
            torch.cuda.synchronize()
            return round(e0.elapsed_time(e1) / args.steps, 5)

        res = {"eager": {"forward": [], "inverse": []}, "graph": {"forward": [], "inverse": []}}
        for _ in range(2):
            for d, fn in (("forward", fwd), ("inverse", inv)):
                res["eager"][d].append(window(lambda: fn(stream)))
                res["graph"][d].append(window(graphs[d].replay))
        plan.wait()
        print(json.dumps({"shape": [n, n, n], "prec": args.prec, "steps": args.steps, "ms_per_transform": res,
                          "launches_per_exec": plan.lastLaunchCount(), "replay_equals_eager": identical, "gpu": gpu}), flush=True)
        del graphs
        plan.destroy()
        del x, out, back
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
