"""Plans with strides (dfft_plan_set_strides) on one GPU (one-rank slab) against the pack / unpack route callers take without
them.

    python tools/embedded_bench.py [--n 512] [--halo 2] [--steps 5] [--rounds 3] [--cases c2c,r2c,dct]

For each case (C2C, R2C / C2R and DCT, f64, n^3 with `halo` ghost layers on every side of the physical field), three arms
run one forward + inverse pair per step:
  (a) dense:    the plan without strides on dense tensors (the reference point: no ghost layers at all);
  (b) pack:     dense.copy_(A[h:-h, h:-h, h:-h]), the dense plan's forward and inverse, A[h:-h, h:-h, h:-h].copy_(back) —
                what a caller with ghost layers does without strides;
  (c) embedded: the plan with in_strides of A, forward from A's interior, inverse back into it (the spectrum dense).
Windows of `steps` pairs alternate between the arms on one stream after a warm-up of each, `rounds` times, timed with CUDA
events (best window reported, ms per pair).  The step timer of one timed forward exec of each plan gives the x pass's time,
which the embedded plan runs with its y-z rows split into a1 = y rows and b = z columns.  Prints one JSON line per case with
the GPU's name, power limit and maximum SM clock read in the same run.  Nothing is gated on the numbers.
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


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def x_pass_ms(plan, fwd):
    """the forward x pass's time from the step timer of one timed exec"""
    plan.enableTimer(True)
    fwd()
    torch.cuda.synchronize()
    steps = plan.stepTimes()
    plan.enableTimer(False)
    return round(sum(ms for label, ms in steps if label.startswith("x pass")), 4)


def run_case(name, n, h, steps, rounds):
    transform, phys_t, spec_t = {"c2c": ("c2c", torch.complex128, torch.complex128), "r2c": ("r2c", torch.float64, torch.complex128),
                                 "dct": ("dct", torch.float64, torch.float64)}[name]
    shape = (n, n, n)
    dense = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform=transform)
    dense.initFFT(dfft.GlobalSize(*shape), None, True)
    A = torch.randn([v + 2 * h for v in shape], dtype=phys_t, device="cuda")
    inner = A[h:-h, h:-h, h:-h]
    emb = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform=transform)
    emb.initFFT(dfft.GlobalSize(*shape), None, True, in_strides=(A.shape[0] * A.stride(0), A.stride(0), A.stride(1)))
    x = inner.contiguous()
    X = torch.empty(dense.getOutSize(), dtype=spec_t, device="cuda")
    back = torch.empty_like(x)

    def fwd(p, o, i):
        if name == "c2c":
            p.execC2C(o, i, dfft.FORWARD, stream=torch.cuda.current_stream())
        elif name == "r2c":
            p.execR2C(o, i, stream=torch.cuda.current_stream())
        else:
            p.execR2R(o, i, dfft.FORWARD, stream=torch.cuda.current_stream())

    def inv(p, o, i):
        if name == "c2c":
            p.execC2C(o, i, dfft.INVERSE, stream=torch.cuda.current_stream())
        elif name == "r2c":
            p.execC2R(o, i, stream=torch.cuda.current_stream())
        else:
            p.execR2R(o, i, dfft.INVERSE, stream=torch.cuda.current_stream())

    def arm_dense():
        fwd(dense, X, x)
        inv(dense, back, X)

    def arm_pack():
        x.copy_(inner)
        fwd(dense, X, x)
        inv(dense, back, X)
        inner.copy_(back)

    def arm_embedded():
        fwd(emb, X, inner)
        inv(emb, inner, X)

    arms = {"dense": arm_dense, "pack": arm_pack, "embedded": arm_embedded}
    for fn in arms.values():  # warm-up: tables, kernel attributes, allocations
        fn(); fn()
    torch.cuda.synchronize()
    best = {k: float("inf") for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            best[k] = min(best[k], timed(fn, steps))
    res = {"case": f"{name} f64 {n}^3 halo {h}", "ms_per_pair": {k: round(v, 4) for k, v in best.items()},
           "embedded_over_pack": round(best["pack"] / best["embedded"], 3),
           "x_pass_ms": {"dense": x_pass_ms(dense, lambda: fwd(dense, X, x)),
                         "embedded": x_pass_ms(emb, lambda: fwd(emb, X, inner))}}
    dense.destroy()
    emb.destroy()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--halo", type=int, default=2)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--cases", default="c2c,r2c,dct")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("embedded_bench.py measures on a GPU; none is visible")
    gpu = gpu_identity()
    for name in a.cases.split(","):
        r = run_case(name, a.n, a.halo, a.steps, a.rounds)
        r["gpu"] = gpu
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
