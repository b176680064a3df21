"""Padded plans against the caller's own padding on one GPU.

At 512^3 with K = 341 per axis (|k| <= 170, the 2/3 rule), f64 and f32, C2C and R2C / C2R, it times
  * the padded plan's forward and inverse (dfft_plan_create_padded), and their passes from the step timer;
  * the ordinary 512^3 plan with the caller's truncation gather after the forward and zero-embedding before the inverse,
    both done with torch indexing;
  * the HBM-byte floor of each at 3.35 TB/s (the H100 SXM data sheet), from the bytes every pass must read and write.
The two paths run in alternating windows of CUDA-event-timed execs, and the card's name and power limit are read in the same
run.  A report, not a gate: it prints one JSON line per case (and writes them to --out).

    python tools/padded_bench.py [--n 512] [--k 341] [--reps 20] [--windows 5] [--out padded_bench.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def floors(n, k, es, r2c):
    """least HBM bytes of the forward (= inverse) of each path: every pass reads and writes its arrays once"""
    nzc, kzc = (n // 2 + 1, k // 2 + 1) if r2c else (n, k)
    real = es // 2 if r2c else es  # the physical side of R2C is real
    z_in = n * n * n * real
    padded = (z_in + n * n * kzc * es) + (n * n * kzc + n * k * kzc) * es + (n * k * kzc + k * k * kzc) * es  # z, y, x passes
    ordinary = (z_in + n * n * nzc * es) + 2 * (2 * n * n * nzc * es)
    gather = 2 * k * k * kzc * es  # read the kept modes, write the K spectrum (the embedding also zeroes the N spectrum)
    return padded, ordinary + gather


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--k", type=int, default=341)
    ap.add_argument("--reps", type=int, default=20, help="execs per timed window")
    ap.add_argument("--windows", type=int, default=5, help="alternating windows per path")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    import distributedfft_b200 as dfft

    if not torch.cuda.is_available():
        raise SystemExit("padded_bench.py needs a CUDA device")
    n, k = args.n, args.k
    dev = "cuda"
    info = card()
    results = []
    for prec in ("double", "float"):
        for transform in ("c2c", "r2c"):
            r2c = transform == "r2c"
            cdt = torch.complex128 if prec == "double" else torch.complex64
            rdt = torch.float64 if prec == "double" else torch.float32
            es = 16 if prec == "double" else 8
            pad = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=prec, transform=transform)
            pad.initFFT(dfft.GlobalSize(n, n, n), None, True, spectral=(k, k, k))
            ordp = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=prec, transform=transform)
            ordp.initFFT(dfft.GlobalSize(n, n, n), None, True)
            g = torch.Generator(device=dev).manual_seed(1)
            x = torch.randn((n, n, n), generator=g, dtype=rdt, device=dev)
            if not r2c:
                x = torch.complex(x, torch.randn((n, n, n), generator=g, dtype=rdt, device=dev))
            kz = k // 2 + 1 if r2c else k
            spec = torch.empty((k, k, kz), dtype=cdt, device=dev)
            full = torch.empty(tuple(ordp.getOutSize()), dtype=cdt, device=dev)
            back = torch.empty_like(x)
            pos = torch.fft.fftfreq(k, 1.0 / k, device=dev).to(torch.long) % n
            pz = torch.arange(kz, device=dev) if r2c else pos
            ix, iy, iz = pos[:, None, None], pos[None, :, None], pz[None, None, :]

            def pad_fwd():
                pad.execR2C(spec, x) if r2c else pad.execC2C(spec, x, dfft.FORWARD)

            def pad_inv():
                pad.execC2R(back, spec) if r2c else pad.execC2C(back, spec, dfft.INVERSE)

            def ord_fwd():
                ordp.execR2C(full, x) if r2c else ordp.execC2C(full, x, dfft.FORWARD)
                spec.copy_(full[ix, iy, iz])

            def ord_inv():
                full.zero_()
                full[ix, iy, iz] = spec
                ordp.execC2R(back, full) if r2c else ordp.execC2C(back, full, dfft.INVERSE)

            def window(fn):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / args.reps

            fns = {"padded_fwd": pad_fwd, "ordinary_fwd_gather": ord_fwd, "padded_inv": pad_inv, "ordinary_embed_inv": ord_inv}
            for fn in fns.values():  # warm-up: modules, tables, torch's indexing kernels
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            times = {name: [] for name in fns}
            for _ in range(args.windows):
                for name, fn in fns.items():
                    times[name].append(window(fn))
            # whether the padded spectrum equals the gathered one bit for bit
            pad_fwd()
            s_pad = spec.clone()
            ord_fwd()
            same_fwd = bool(torch.equal(s_pad, spec))
            steps = {}
            pad.enableTimer(True)
            for name, fn in (("fwd", pad_fwd), ("inv", pad_inv)):
                fn()
                torch.cuda.synchronize()
                steps[name] = [(label, round(ms, 4)) for label, ms in pad.stepTimes()]
            pad.enableTimer(False)
            fp, fo = floors(n, k, es, r2c)
            med = {name: sorted(v)[len(v) // 2] for name, v in times.items()}
            res = {"card": info, "n": n, "k": k, "precision": prec, "transform": transform, "ms_median": {a: round(b, 4) for a, b in med.items()},
                   "ms_windows": {a: [round(t, 4) for t in b] for a, b in times.items()}, "padded_steps_ms": steps,
                   "floor_ms": {"padded": round(fp / HBM_BYTES_PER_S * 1e3, 4), "ordinary_plus_gather": round(fo / HBM_BYTES_PER_S * 1e3, 4)},
                   "speedup_fwd": round(med["ordinary_fwd_gather"] / med["padded_fwd"], 3),
                   "speedup_inv": round(med["ordinary_embed_inv"] / med["padded_inv"], 3), "forward_bit_identical": same_fwd}
            print(json.dumps(res), flush=True)
            results.append(res)
            pad.destroy()
            ordp.destroy()
            del x, spec, full, back
            torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
