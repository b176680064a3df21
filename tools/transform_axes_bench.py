"""Kept axes on one GPU (one-rank slab, C2C): the full transform against plans with x, y or z kept.

    python tools/transform_axes_bench.py [--steps 20] [--rounds 3] [--n 512] [--precs f64,f32]

Plans, side by side for each precision: full (every axis), x_kept, y_kept and z_kept, each forward and inverse.  Windows
of `steps` execs alternate between the plans on one stream, `rounds` times, timed with CUDA events (best window
reported).  One timed exec per plan and direction gives the per-step times (the step timer).

"copy_vs_fft" sets each copy step against the FFT pass over the same views.  On one GPU the only copy is a kept y, and
the slab plan's full exec fuses z and y into one stage at this size, so the reference is a pencil 1 x 1 plan: its full
exec runs a standalone y pass, and its y_kept exec a y copy, over the same blocked hand-over views.  The script checks
that with dfft_plan_describe (lengths, extents and strides of both views of both steps) and reports "same_views".
Prints one JSON line per precision, with the GPU's name, power limit and maximum SM clock read in the same run.  Nothing is
gated on the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import distributedfft_b200 as dfft  # noqa: E402
from distributedfft_b200._lib import check, lib  # noqa: E402

MASKS = {"full": None, "x_kept": (False, True, True), "y_kept": (True, False, True), "z_kept": (True, True, False)}


def gpu_identity():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
    name, power, clock = [v.strip() for v in r.stdout.strip().split(",")]
    return {"name": name, "power_limit_w": float(power), "sm_max_mhz": float(clock)}


def describe(plan, inverse):
    need = C.c_size_t()
    check(lib().dfft_plan_describe(plan._h, inverse, 3, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib().dfft_plan_describe(plan._h, inverse, 3, buf, need.value, C.byref(need)))
    return json.loads(buf.value.decode())


def view_shape(st):
    """a pass step's geometry without its base addresses"""
    def v(view):
        return view["nseg"], view["sN"], [(g["sA0"], g["sA1"], g["n0"]) for g in view["segs"]]
    return st.get("n", 1 << st["log2n"]), st["A0"], st["A1"], st["B"], v(st["in"]), v(st["out"])


def run(n, prec, steps, rounds, gpu):
    shape = (n, n, n)
    pname = "double" if prec == "f64" else "float"
    cdt = torch.complex128 if prec == "f64" else torch.complex64
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.complex(torch.rand(shape, generator=g, device="cuda"), torch.rand(shape, generator=g, device="cuda")).to(cdt)
    y, z = torch.empty_like(x), torch.empty_like(x)
    plans = {}
    for t, axes in MASKS.items():
        p = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=pname, transform="c2c")
        p.initFFT(dfft.GlobalSize(*shape), None, True, transform_axes=axes)
        plans[t] = p
    for t, axes in (("pencil_full", None), ("pencil_y_kept", MASKS["y_kept"])):
        p = dfft.MPIcuFFT_Pencil(dfft.Configurations(), dfft.Comm(), precision=pname, transform="c2c")
        p.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1), True, transform_axes=axes)
        plans[t] = p
    stream = torch.cuda.current_stream()

    def ex(t, inverse):
        # inverse execs read the forward output y and write z; forward execs read x and write y
        if inverse:
            plans[t].execC2C(z, y, dfft.INVERSE, stream=stream)
        else:
            plans[t].execC2C(y, x, dfft.FORWARD, stream=stream)

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

    ms = {f"{t}_{d}": [] for t in plans for d in ("fwd", "inv")}
    for _ in range(rounds):
        for t in plans:
            for d, inv in (("fwd", False), ("inv", True)):
                ms[f"{t}_{d}"].append(round(window(t, inv), 5))
    # per-step times: the median of `rounds` timed execs per plan and direction
    steps_ms = {}
    for t, p in plans.items():
        p.enableTimer(True)
        for d, inv in (("fwd", False), ("inv", True)):
            runs = []
            for _ in range(rounds):
                ex(t, inv)
                p.wait()
                runs.append(p.stepTimes())
            steps_ms[f"{t}_{d}"] = [(runs[0][i][0], round(sorted(r[i][1] for r in runs)[len(runs) // 2], 5)) for i in range(len(runs[0]))]
        p.enableTimer(False)
    best = {k: min(v) for k, v in ms.items()}
    copy_vs_fft = {}
    for d, inv in (("fwd", 0), ("inv", 1)):
        kept = [s_ for s_ in describe(plans["pencil_y_kept"], inv)["steps"] if s_["type"] == 0]
        full = [s_ for s_ in describe(plans["pencil_full"], inv)["steps"] if s_["type"] == 0]
        for st in kept:
            if st["kind"] not in (6, 7):
                continue
            ref = [j for j, f in enumerate(full) if f["label"] == st["label"].replace("copy", "pass")]
            same = bool(ref) and view_shape(full[ref[0]]) == view_shape(st)
            copy_vs_fft[f"pencil {d}: {st['label']}"] = {
                "copy_ms": dict(steps_ms[f"pencil_y_kept_{d}"])[st["label"]],
                "fft_pass_ms": dict(steps_ms[f"pencil_full_{d}"])[full[ref[0]]["label"]] if ref else None,
                "same_views": same, "A0_A1_B": [st["A0"], st["A1"], st["B"]]}
    print(json.dumps({"shape": list(shape), "prec": prec, "steps": steps, "ms": ms, "best_ms": best, "step_ms": steps_ms,
                      "copy_vs_fft": copy_vs_fft,
                      "x_kept_over_full": {d: round(best[f"x_kept_{d}"] / best[f"full_{d}"], 4) for d in ("fwd", "inv")}, "gpu": gpu}), flush=True)
    for p in plans.values():
        p.destroy()
    del x, y, z
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--precs", default="f64,f32")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("transform_axes_bench.py needs a GPU")
    gpu = gpu_identity()
    for prec in args.precs.split(","):
        run(args.n, prec, args.steps, args.rounds, gpu)


if __name__ == "__main__":
    main()
