"""Batched 3D transforms on one GPU: one batched exec against a loop of the unbatched plan and against cuFFT batched.

    python tools/batch_bench.py [--workloads 64:f64:64,128:f64:16] [--steps 20] [--warmup 3] [--out DIR]

A workload is N:precision:batch, one-rank slab complex fields of N^3 points, forward.  For each one, in alternating
windows of `steps` execs on one stream, CUDA events time:
  batched/eager   one exec of a plan created with the batch (dfft_plan_create_batched);
  batched/graph   a replay of a CUDA graph holding that exec;
  loop/eager      one exec of the unbatched plan per field;
  loop/graph      a replay of a graph holding that loop (the fastest loop a caller can build without batching);
  cufft           cufftPlanMany (rank 3) over the same fields (tools/cufft_many_ref.cu, compiled here into a temporary
                  directory).
Reported per workload: ms per exec and per field, the HBM floor (one read and one write of every field at the 3.35 TB/s of
the H100 SXM data sheet) and its ratio to the batched graph replay, the launches per exec, and whether the batched
output equals the per-field output bit for bit.  The GPU's name, power limit and maximum SM clock are read in the same
run.  Prints one JSON line per workload (and writes them to DIR/batch_bench.jsonl with --out).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import distributedfft_b200 as dfft  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
DEFAULT = "64:f64:2,64:f64:8,64:f64:64,64:f64:256,32:f64:2,32:f64:512,64:f32:64,128:f64:16,256:f64:4"


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def cufft_many(tmpdir):
    """tools/cufft_many_ref.cu built into tmpdir; returns the loaded library"""
    so = os.path.join(tmpdir, "libcufft_many_ref.so")
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                    os.path.join(ROOT, "tools", "cufft_many_ref.cu"), "-lcufft", "-o", so], check=True)
    lib = C.CDLL(so)
    lib.cufft_ref_3d_many.restype = C.c_int
    lib.cufft_ref_3d_many.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int]
    return lib


def plan_of(n, f64, batch):
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform="c2c")
    plan.initFFT(dfft.GlobalSize(n, n, n), None, True, batch=batch)
    return plan


def run(n, f64, batch, steps, warmup, ref_lib, gpu):
    rdt = torch.float64 if f64 else torch.float32
    stream = torch.cuda.current_stream()
    g = torch.Generator(device="cuda").manual_seed(1234)
    x = torch.complex(torch.rand((batch, n, n, n), generator=g, device="cuda", dtype=rdt) * 255,
                      torch.rand((batch, n, n, n), generator=g, device="cuda", dtype=rdt) * 255)
    out_b, out_l, out_c = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    pb, p1 = plan_of(n, f64, batch), plan_of(n, f64, 1)

    def batched(s):
        pb.execC2C(out_b, x, dfft.FORWARD, stream=s)

    def loop(s):
        for f in range(batch):
            p1.execC2C(out_l[f], x[f], dfft.FORWARD, stream=s)

    for _ in range(warmup):
        batched(stream)
        loop(stream)
    pb.wait()
    p1.wait()
    launches = pb.lastLaunchCount()
    identical = bool(torch.equal(out_b, out_l))
    graphs = {}
    for name, fn in (("batched", batched), ("loop", loop)):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr):
            fn(torch.cuda.current_stream())
        gr.replay()
        graphs[name] = gr
    torch.cuda.synchronize()

    def window(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps

    def cufft_window():
        ms = C.c_float()
        rc = ref_lib.cufft_ref_3d_many(1 if f64 else 0, 0, n, n, n, batch, out_c.data_ptr(), x.data_ptr(), C.byref(ms), steps)
        assert rc == 0, rc
        return ms.value

    res = {k: [] for k in ("batched/eager", "batched/graph", "loop/eager", "loop/graph", "cufft")}
    for _ in range(3):
        res["batched/eager"].append(window(lambda: batched(stream)))
        res["batched/graph"].append(window(graphs["batched"].replay))
        res["loop/eager"].append(window(lambda: loop(stream)))
        res["loop/graph"].append(window(graphs["loop"].replay))
        res["cufft"].append(cufft_window())
    pb.wait()
    best = {k: min(v) for k, v in res.items()}
    field_bytes = n ** 3 * (16 if f64 else 8)
    floor_ms = 2 * batch * field_bytes / HBM_BYTES_PER_S * 1e3
    line = {"shape": [n, n, n], "prec": "f64" if f64 else "f32", "batch": batch, "steps": steps,
            "path": "one launch" if launches == 1 else "per field", "launches_per_exec": launches,
            "ms_per_exec": {k: [round(t, 5) for t in v] for k, v in res.items()},
            "ms_per_field_best": {k: round(v / batch, 6) for k, v in best.items()},
            "hbm_floor_ms": round(floor_ms, 5), "floor_over_batched_graph": round(floor_ms / best["batched/graph"], 3),
            "batched_over_loop_graph": round(best["batched/graph"] / best["loop/graph"], 3),
            "batched_equals_loop": identical, "gpu": gpu}
    del graphs
    pb.destroy()
    p1.destroy()
    del x, out_b, out_l, out_c
    torch.cuda.empty_cache()
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=DEFAULT)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = gpu_identity()
    with tempfile.TemporaryDirectory() as td:
        ref_lib = cufft_many(td)
        lines = []
        for w in args.workloads.split(","):
            n, prec, b = w.split(":")
            line = run(int(n), prec == "f64", int(b), args.steps, args.warmup, ref_lib, gpu)
            print(json.dumps(line), flush=True)
            lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_bench.jsonl"), "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
