"""Per-item timeline of the fused z + y stage (fft_zy_fused_kernel / fft_zy_fed_kernel), from the trace build.

    python tools/zy_trace.py [--n 512] [--lib PATH] [--feeds 1,0] [--out DIR]

Builds the library with -DDFFT_ZY_TRACE into a temporary directory (or takes --lib) and loads it through DFFT_LIB.  Thread 0
of every CTA then writes %globaltimer stamps per work item (ZyStamp in fft_kernels.cuh): ticket read, dependency met, inputs
landed (fed kernel), first exchange done, last gather done, stores issued, item done.  For an n^3 complex-double slab plan,
forward and inverse, once per feed (DFFT_ZY_FEED=1 fed, 0 register-fed: the kernel of the builds before the fed one),
after two warm-up execs, one traced exec is read back and reported:
  * per phase (A / B), the median and p90 of each interval, in microseconds;
  * the dependency waits: the share of all CTA time spent between ticket and dependency met (it includes thread 0's
    wait for the next ticket's atomic draw, about 0.8 us per item on an H100), and the phase-B items above 1 us;
  * the stage time (first ticket to last item done) and the achieved rates: HBM = one read + one write of the array,
    L2 = that plus the intermediate written and read once more (4 array-sizes through the L2), both over the stage time.
The stamps cost a few instructions of thread 0 per item, so the traced stage runs slightly slower than the untraced one.
"""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SLOTS = 8
TICKET, DEP, INPUTS, EXCH, LAST, STORED, DONE, WHERE = range(SLOTS)
INTERVALS = [("dependency wait", TICKET, DEP), ("inputs landed", DEP, INPUTS), ("to first exchange", DEP, EXCH),
             ("first exchange -> last gather", EXCH, LAST), ("last gather -> stores issued", LAST, STORED),
             ("stores -> done", STORED, DONE), ("item (ticket -> done)", TICKET, DONE)]


def build_variant(tmp):
    from distributedfft_b200 import build as b

    return b.build(defines=["-DDFFT_ZY_TRACE"], out=os.path.join(tmp, "libdfft_zy_trace.so"), objdir=os.path.join(tmp, "obj"))


def pct(v, q):
    import numpy as np

    return float(np.percentile(v, q)) if len(v) else float("nan")


def analyse(tr, n, fed=True):
    import numpy as np

    t = tr.astype(np.int64)
    phase = (tr[:, WHERE] & 1).astype(int)
    cta = ((tr[:, WHERE] & 0xffffffff) >> 1).astype(int)
    t0 = t[:, TICKET].min()
    stage_ns = float(t[:, DONE].max() - t0)
    res = {"items": int(len(t)), "ctas": int(cta.max() + 1), "stage_ms": stage_ns / 1e6}
    nz = np.diff(np.unique(t[:, TICKET]))
    res["timer_resolution_ns"] = int(nz[nz > 0].min()) if (nz > 0).any() else None
    for ph, name in ((0, "A"), (1, "B")):
        m = phase == ph
        rows = {}
        for label, a, b in INTERVALS:
            if not fed and INPUTS in (a, b):
                continue  # register-fed: no copy to wait for (the slot holds an earlier fed launch's stamps, if any)
            d = (t[m, b] - t[m, a]) / 1e3
            rows[label] = {"median_us": round(pct(d, 50), 3), "p90_us": round(pct(d, 90), 3)}
        res["phase_" + name] = rows
    # between items of one CTA: item done -> next ticket read (draw, barrier, ticket decode)
    order = np.lexsort((t[:, TICKET], cta))
    tc, cc = t[order], cta[order]
    same = cc[1:] == cc[:-1]
    gap = (tc[1:, TICKET] - tc[:-1, DONE])[same] / 1e3
    res["between items"] = {"median_us": round(pct(gap, 50), 3), "p90_us": round(pct(gap, 90), 3)}
    dep = (t[:, DEP] - t[:, TICKET]).astype(float)
    busy = float((t[:, DONE] - t[:, TICKET]).sum())
    res["dependency_wait_share"] = round(float(dep.sum()) / busy, 4) if busy > 0 else None
    res["items_waiting_over_1us"] = int((dep[phase == 1] > 1000).sum())
    bytes_arr = 16.0 * n ** 3
    res["hbm_TBps"] = round(2 * bytes_arr / stage_ns / 1e3, 3)
    res["l2_TBps"] = round(4 * bytes_arr / stage_ns / 1e3, 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=512)
    ap.add_argument("--lib", default=None, help="an already built trace variant")
    ap.add_argument("--feeds", default="1,0")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="zy_trace_")
    path = args.lib or build_variant(tmp)
    os.environ["DFFT_LIB"] = path
    from distributedfft_b200 import _lib

    _lib.LIB_PATH = path
    import numpy as np
    import torch

    import distributedfft_b200 as dfft

    raw = _lib.lib()
    raw.dfft_zy_trace_copy.restype = C.c_int
    raw.dfft_zy_trace_copy.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t]
    props = torch.cuda.get_device_properties(0)
    import subprocess

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"# {props.name}; nvidia-smi: {smi}; lib {path}")
    n = args.n
    shape = (n, n, n)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=torch.float64), torch.rand(shape, generator=g, device="cuda", dtype=torch.float64))
    out = torch.empty_like(x)
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="c2c")
    plan.initFFT(dfft.GlobalSize(*shape), None, True)
    items = 2 * n * (n * n // 4096)
    buf = np.zeros((items, SLOTS), dtype=np.uint64)
    report = {"gpu": smi, "n": n}
    for feed in [int(v) for v in args.feeds.split(",")]:
        os.environ["DFFT_ZY_FEED"] = str(feed)
        for direction, dname in ((dfft.FORWARD, "forward"), (dfft.INVERSE, "inverse")):
            for _ in range(3):
                plan.execC2C(out, x, direction)
            torch.cuda.synchronize()
            got = raw.dfft_zy_trace_copy(plan._h, 1 if direction == dfft.INVERSE else 0, buf.ctypes.data, buf.nbytes)
            if got != items:
                raise RuntimeError(f"dfft_zy_trace_copy returned {got}, expected {items}")
            r = analyse(buf.copy(), n, fed=bool(feed))
            key = f"{'fed' if feed else 'register-fed'} {dname}"
            report[key] = r
            print(f"\n== {key}: stage {r['stage_ms']:.3f} ms, HBM {r['hbm_TBps']} TB/s, L2 {r['l2_TBps']} TB/s, "
                  f"dependency waits {100 * r['dependency_wait_share']:.2f} % of CTA time "
                  f"({r['items_waiting_over_1us']} B items > 1 us), timer step {r['timer_resolution_ns']} ns, {r['ctas']} CTAs")
            for ph in ("A", "B"):
                for label, v in r["phase_" + ph].items():
                    print(f"  {ph}  {label:32s} median {v['median_us']:8.3f} us   p90 {v['p90_us']:8.3f} us")
            print(f"     {'between items':32s} median {r['between items']['median_us']:8.3f} us   p90 {r['between items']['p90_us']:8.3f} us")
    os.environ.pop("DFFT_ZY_FEED", None)
    plan.destroy()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "zy_trace.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
