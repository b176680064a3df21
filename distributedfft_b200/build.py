"""Build libdfft.so (sm_90a) in-tree with nvcc.  `python -m distributedfft_b200.build` or build.build().

The kernel instantiations (one translation unit per precision x log2 length, and per 16-bit format x log2 length) are
compiled in parallel;
objects are cached under distributedfft_b200/csrc/build/ keyed by source mtimes.
"""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "build")
LIB = os.path.join(HERE, "libdfft.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--threads", "1"]
MAX_LOG2N = 13


def _stamp(paths):
    h = hashlib.sha1()
    for p in sorted(paths):
        st = os.stat(p)
        h.update(f"{p}:{st.st_mtime_ns}:{st.st_size}".encode())
    return h.hexdigest()


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return r.stdout + r.stderr


def _flags_key():
    # the compiler and its flags belong to a build product as much as its sources: a new target architecture must not
    # reuse objects compiled for another one
    return "|".join([NVCC, *ARCH, *COMMON])


def _compile(src, obj, defs, deps, verbose):
    stamp = _stamp(deps) + "|" + " ".join(defs) + "|" + _flags_key()
    sfile = obj + ".stamp"
    if os.path.exists(obj) and os.path.exists(sfile) and open(sfile).read() == stamp:
        return obj
    cmd = [NVCC, *ARCH, *COMMON, *defs, "-c", src, "-o", obj]
    out = _run(cmd)
    if verbose and out.strip():
        print(out)
    with open(sfile, "w") as f:
        f.write(stamp)
    return obj


def build(verbose: bool = False, force: bool = False, defines=(), out: str = LIB, objdir: str = OBJ) -> str:
    """defines / out / objdir: experimental variants (e.g. build(defines=["-DDFFT_CONTIG_THREADS=128"],
    out=".../libdfft_t128.so", objdir=".../build_t128"); select at run time with DFFT_LIB=<path>)."""
    OBJ_ = objdir
    os.makedirs(OBJ_, exist_ok=True)
    headers = [os.path.join(CSRC, h) for h in ("fft_core.cuh", "fft_kernels.cuh", "zy_order.hpp", "geometry.hpp", "bluestein.hpp", "r2r.hpp")]
    headers.append(os.path.join(HERE, "..", "include", "dfft.h"))
    jobs = []
    inst = os.path.join(CSRC, "fft_inst.cu")
    for tname in ("double", "float"):
        for l in range(1, MAX_LOG2N + 1):
            obj = os.path.join(OBJ_, f"fft_inst_{tname}_{l}.o")
            jobs.append((inst, obj, [f"-DDFFT_T={tname}", f"-DDFFT_LOG2N={l}", *defines], [inst, *headers]))
    # the passes of 16-bit plans: f32 arithmetic, one unit per stored format and length
    for sname, stype in (("half", "__half"), ("bf16", "__nv_bfloat16")):
        for l in range(1, MAX_LOG2N + 1):
            obj = os.path.join(OBJ_, f"fft_inst_{sname}_{l}.o")
            jobs.append((inst, obj, ["-DDFFT_T=float", f"-DDFFT_S={stype}", f"-DDFFT_LOG2N={l}", *defines], [inst, *headers]))
    for name in ("fft_dispatch.cu", "dfft_plan.cu"):
        src = os.path.join(CSRC, name)
        jobs.append((src, os.path.join(OBJ_, name.replace(".cu", ".o")), list(defines), [src, *headers]))
    if force:
        for _, obj, _, _ in jobs:
            if os.path.exists(obj + ".stamp"):
                os.remove(obj + ".stamp")
    workers = max(1, min(len(jobs), (os.cpu_count() or 2)))
    objs = []
    with cf.ThreadPoolExecutor(workers) as ex:
        futs = [ex.submit(_compile, s, o, d, deps, verbose) for s, o, d, deps in jobs]
        for f in futs:
            objs.append(f.result())
    lstamp = _stamp(objs) + "|" + _flags_key()
    lfile = out + ".stamp"
    if not (os.path.exists(out) and os.path.exists(lfile) and open(lfile).read() == lstamp):
        tmp = out + ".tmp"
        cmd = [NVCC, *ARCH, "-shared", "-o", tmp, *objs, "-lnccl", "-Xlinker", "-z,noexecstack"]
        _run(cmd)
        os.replace(tmp, out)  # atomic: a snapshot of the tree never sees a half-written library
        with open(lfile, "w") as f:
            f.write(lstamp)
    return out


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
