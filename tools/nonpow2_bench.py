"""One-rank C2C plans with axis lengths that are not powers of two (Bluestein passes) on one GPU, next to the 512^3
power-of-two plan and single-GPU cuFFT (oracle/cufft_ref.cu, cufftPlan3d) at the same shapes.

    python tools/nonpow2_bench.py [--steps 10] [--rounds 3] [--cases all|name,name]

Per case: forward execs in `rounds` windows of `steps` execs on one stream, timed with CUDA events (the best window is
reported), then one timed exec with the plan's step timer for the per-pass times, then cuFFT's time per exec for the same
shape and precision (built into a temporary directory).  Prints one JSON line per case with the GPU's name, power limit
and maximum SM clock, read in the same run.
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

CASES = {
    # name: (shape, f64)
    "c2c_384_f64": ((384, 384, 384), True),
    "c2c_500_f64": ((500, 500, 500), True),
    "c2c_768_f64": ((768, 768, 768), True),
    "c2c_384_f32": ((384, 384, 384), False),
    "c2c_512_f64": ((512, 512, 512), True),
}


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def cufft_ref(tmpdir):
    so = os.path.join(tmpdir, "libcufft_ref.so")
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                    os.path.join(ROOT, "oracle", "cufft_ref.cu"), "-lcufft", "-o", so], check=True)
    lib = C.CDLL(so)
    lib.cufft_ref_3d.restype = C.c_int
    lib.cufft_ref_3d.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int]
    return lib


def run_case(name, steps, rounds, gpu, ref):
    shape, f64 = CASES[name]
    rdt = torch.float64 if f64 else torch.float32
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform="c2c")
    plan.initFFT(dfft.GlobalSize(*shape), None, True)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
    out = torch.empty_like(x)
    stream = torch.cuda.current_stream()
    for _ in range(3):
        plan.execC2C(out, x, dfft.FORWARD, stream=stream)
    windows = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            plan.execC2C(out, x, dfft.FORWARD, stream=stream)
        e1.record()
        e1.synchronize()
        windows.append(e0.elapsed_time(e1) / steps)
    plan.enableTimer(True)
    plan.execC2C(out, x, dfft.FORWARD)
    torch.cuda.synchronize()
    passes = plan.stepTimes()
    plan.enableTimer(False)
    ms = C.c_float()
    ref_out = torch.empty_like(x)
    assert ref.cufft_ref_3d(1 if f64 else 0, 0, *shape, ref_out.data_ptr(), x.data_ptr(), C.byref(ms), steps) == 0
    rel = float((out - ref_out).abs().pow(2).sum().sqrt() / ref_out.abs().pow(2).sum().sqrt())
    plan.destroy()
    del x, out, ref_out
    torch.cuda.empty_cache()
    return {"case": name, "shape": list(shape), "precision": "f64" if f64 else "f32", "ms_per_exec": round(min(windows), 4),
            "windows_ms": [round(w, 4) for w in windows], "passes_ms": [[label, round(t, 4)] for label, t in passes],
            "cufft_ms": round(ms.value, 4), "rel_l2_vs_cufft": rel, "gpu": gpu}


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cases", default="all")
    a = ap.parse_args(argv)
    names = list(CASES) if a.cases == "all" else a.cases.split(",")
    gpu = gpu_identity()
    with tempfile.TemporaryDirectory() as td:
        ref = cufft_ref(td)
        for name in names:
            print(json.dumps(run_case(name, a.steps, a.rounds, gpu, ref)), flush=True)


if __name__ == "__main__":
    main()
