"""In-place against out-of-place plans on one GPU: time per forward + inverse pair, work area and memory footprint.

    python tools/inplace_bench.py [--steps 20] [--rounds 3] [--cases all|name,name]

Cases: 512^3 and 256^3 complex-double, 1024^3 R2C / C2R f64, 64 fields of 64^3 complex-double (one launch).  Both plans of
a case exist side by side; their windows of `steps` forward + inverse pairs (inverse scale 1/N, so that the in-place
buffer keeps its magnitude) alternate on one stream, `rounds` times, timed with CUDA events.  Prints one JSON line per
case: ms per pair of every window, the work area and the bytes each variant holds (caller buffers + work area), the
device's free memory with both allocated, and the GPU's name, power limit and maximum SM clock, read in the same run.
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
    # name: (shape, transform, batch)
    "c2c_512": ((512, 512, 512), "c2c", 1),
    "c2c_256": ((256, 256, 256), "c2c", 1),
    "r2c_1024": ((1024, 1024, 1024), "r2c", 1),
    "c2c_64x64": ((64, 64, 64), "c2c", 64),
}


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def run_case(name, steps, rounds, gpu):
    shape, transform, batch = CASES[name]
    c2c = transform == "c2c"
    nx, ny, nz = shape
    nzc = nz if c2c else nz // 2 + 1
    plans = {}
    for variant in ("inplace", "out_of_place"):
        p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform=transform)
        p.initFFT(dfft.GlobalSize(*shape), None, True, batch, variant == "inplace")
        p.setScale(1.0, 1.0 / (nx * ny * nz))
        plans[variant] = p
    g = torch.Generator(device="cuda").manual_seed(1)
    real_shape, spec_shape = (batch, nx, ny, nz), (batch, nx, ny, nzc)
    if c2c:
        x = torch.complex(torch.rand(real_shape, generator=g, device="cuda", dtype=torch.float64),
                          torch.rand(real_shape, generator=g, device="cuda", dtype=torch.float64))
    else:
        x = torch.rand(real_shape, generator=g, device="cuda", dtype=torch.float64)
    spec = torch.empty(spec_shape, device="cuda", dtype=torch.complex128)
    buf = torch.empty(spec_shape, device="cuda", dtype=torch.complex128)  # domain size per field
    assert buf[0].numel() * 16 == plans["inplace"].getDomainSize()
    if c2c:
        buf.copy_(x)
        real_side = buf
    else:
        real_side = torch.view_as_real(buf).view(batch, nx, ny, 2 * nzc)  # padded rows
        real_side[..., :nz] = x
    stream = torch.cuda.current_stream()

    def pair(variant):
        p = plans[variant]
        out, back = (buf, buf) if variant == "inplace" else (spec, x)
        src_f, src_i = (real_side, buf) if variant == "inplace" else (x, spec)
        if c2c:
            p.execC2C(out, src_f, dfft.FORWARD, stream=stream)
            p.execC2C(back, src_i, dfft.INVERSE, stream=stream)
        else:
            p.execR2C(out, src_f, stream=stream)
            p.execC2R(real_side if variant == "inplace" else back, src_i, stream=stream)

    def window(variant):
        pair(variant)  # warm-up
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            pair(variant)
        e1.record(stream)
        torch.cuda.synchronize()
        return round(e0.elapsed_time(e1) / steps, 5)

    res = {"inplace": [], "out_of_place": []}
    for _ in range(rounds):
        for variant in res:
            res[variant].append(window(variant))
    for p in plans.values():
        p.wait()
    free, total = torch.cuda.mem_get_info()
    work = {v: plans[v].getWorkSizeDevice() for v in plans}
    held = {"inplace": work["inplace"] + buf.numel() * 16,
            "out_of_place": work["out_of_place"] + x.numel() * x.element_size() + spec.numel() * 16}
    best = {k: min(v) for k, v in res.items()}
    print(json.dumps({"case": name, "shape": list(shape), "batch": batch, "transform": transform, "steps": steps,
                      "ms_per_fwd_inv_pair": res, "best_ms": best, "inplace_over_out_of_place": round(best["inplace"] / best["out_of_place"], 4),
                      "work_bytes": work, "bytes_held": held, "free_bytes_with_both": free, "device_bytes": total, "gpu": gpu}), flush=True)
    for p in plans.values():
        p.destroy()
    del x, spec, buf, real_side
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cases", default="all")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("inplace_bench.py needs a GPU")
    names = list(CASES) if args.cases == "all" else args.cases.split(",")
    gpu = gpu_identity()
    for name in names:
        run_case(name, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
