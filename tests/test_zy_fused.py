"""The fused z + y stage of one-rank slab C2C plans (fft_zy_fused_kernel): its work list, its schedule, and its results
against cuFFT and against the standalone passes."""
import ctypes as C
import os
import subprocess
import tempfile

import pytest

import distributedfft_b200 as dfft
from oracle import dft_oracle as O

from test_schedule_emulation import P2P, SL, SYNC, describe, run_case

HERE = os.path.dirname(os.path.abspath(__file__))


def test_work_list():
    """Every z line and y tile issued once, dependencies on lower tickets only, counter targets over three launches."""
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "zy_order_test")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "zy_order_test.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0 and "fails=0" in r.stdout, r.stdout[-2000:]


def _labels(shape, inverse, prec=dfft.F64):
    sc = describe(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, prec)
    return [s["label"] for s in sc["steps"]]


def test_fused_only_above_the_l2():
    """Geometry-only plans assume an H100's 50 MB L2: 256^3 complex-double (256 MiB) is fused, 128^3 (32 MiB) is not;
    Ny != Nz and R2C keep the separate passes."""
    assert _labels((256, 256, 256), 0) == ["zy pass: z phase", "zy pass: y phase", "x pass"]
    assert _labels((256, 256, 256), 1) == ["x pass", "yz pass: y phase", "yz pass: z phase"]
    assert _labels((128, 128, 128), 0) == ["z pass", "y pass", "x pass"]
    assert _labels((256, 512, 256), 0) == ["z pass", "y pass", "x pass"]
    assert _labels((512, 1024, 1024), 0) == ["z pass", "y pass", "x pass"]  # 1024-point planes: not instantiated
    sc = describe(0, 1, SL, dfft.R2C, (256, 256, 256), 1, 1, P2P, SYNC, 0, 3)
    assert [s["label"] for s in sc["steps"]][0] == "z pass (R2C)"


@pytest.mark.parametrize("inverse", [0, 1])
def test_fused_schedule_replay(inverse):
    """The fused stage's two phases of a 256^3 complex-double plan, replayed on the CPU with the views they use, against
    the oracle."""
    assert run_case(1, SL, dfft.C2C, (256, 256, 256), 1, 1, P2P, SYNC, inverse, 3) < 1e-12


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _cufft_lib():
    path = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "libcufft_ref.so")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/libcufft_ref.so not built")
    lib = C.CDLL(path)
    lib.cufft_ref_3d.restype = C.c_int
    lib.cufft_ref_3d.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int]
    return lib


def _rel_l2(a, b):
    a = a.reshape(-1); b = b.reshape(-1)
    num = den = 0.0
    step = 1 << 26
    for i in range(0, a.numel(), step):
        d = a[i:i + step] - b[i:i + step]
        r = b[i:i + step]
        num += float((d.real.double() ** 2 + d.imag.double() ** 2).sum())
        den += float((r.real.double() ** 2 + r.imag.double() ** 2).sum())
    return (num / den) ** 0.5


def _plan(shape, prec):
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if prec == dfft.F64 else "float", transform="c2c")
    plan.initFFT(dfft.GlobalSize(*shape), None, True)
    return plan


@pytest.mark.gpu
@pytest.mark.parametrize("shape,prec", [((64, 512, 512), dfft.F64), ((1024, 256, 256), dfft.F64), ((512, 512, 512), dfft.F32),
                                        ((64, 512, 512), dfft.F32), ((1024, 256, 256), dfft.F32)])
def test_fused_vs_cufft(shape, prec):
    """Fused plans above the L2 size against cufftPlan3d, forward and inverse."""
    import torch

    lib = _cufft_lib()
    f64 = prec == dfft.F64
    rdt = torch.float64 if f64 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
    plan = _plan(shape, prec)
    out = torch.empty_like(x)
    plan.execC2C(out, x, dfft.FORWARD)
    assert plan.lastLaunchCount() == 2
    ref = torch.empty_like(x)
    ms = C.c_float()
    assert lib.cufft_ref_3d(1 if f64 else 0, 0, *shape, ref.data_ptr(), x.data_ptr(), C.byref(ms), 1) == 0
    tol = O.TOL["f64" if f64 else "f32"]
    assert _rel_l2(out, ref) < tol
    back = torch.empty_like(x)
    plan.execC2C(back, ref, dfft.INVERSE)
    assert plan.lastLaunchCount() == 2
    assert lib.cufft_ref_3d(1 if f64 else 0, 1, *shape, out.data_ptr(), ref.data_ptr(), C.byref(ms), 1) == 0
    assert _rel_l2(back, out) < tol
    # repeated execs, each on a new input into the other output: the fused stage's counters carry over from launch to launch,
    # and a phase-B item that read the previous exec's intermediate would not match
    for r in range(3):
        xr = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
        dst = back if r % 2 == 0 else out
        plan.execC2C(dst, xr, dfft.FORWARD)
        assert plan.lastLaunchCount() == 2
        assert lib.cufft_ref_3d(1 if f64 else 0, 0, *shape, ref.data_ptr(), xr.data_ptr(), C.byref(ms), 1) == 0
        assert _rel_l2(dst, ref) < tol, f"repeated exec {r}"
        del xr
    plan.destroy()
    del x, out, ref, back
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_fused_matches_standalone_passes():
    """512^3 complex-double: the fused plan against the three standalone passes (fft1d_contig / fft1d_strided /
    fft1d_general) on the same input, run in the plan's order (forward z, y, x; inverse x, y, z).  Every line goes through
    the same per-line arithmetic and twiddles, so the results are bit-identical."""
    import torch

    n = 512
    prec = dfft.F64
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.complex(torch.rand((n, n, n), generator=g, device="cuda", dtype=torch.float64) * 255,
                      torch.rand((n, n, n), generator=g, device="cuda", dtype=torch.float64) * 255)
    plan = _plan((n, n, n), prec)
    s = torch.cuda.current_stream()
    for direction in (dfft.FORWARD, dfft.INVERSE):
        out = torch.empty_like(x)
        plan.execC2C(out, x, direction)
        a = torch.empty_like(x)
        b = torch.empty_like(x)
        if direction == dfft.FORWARD:  # z, y, x
            dfft.fft1d_contig(prec, 0, direction, n, n * n, a, n, x, n, s)
            dfft.fft1d_strided(prec, direction, n, n, n, b, a, s)
            dfft.fft1d_general(prec, direction, n, 1, 1, n * n, a, (0, 0, n * n), b, (0, 0, n * n), s)
        else:  # the plan's inverse order: x, y, z
            dfft.fft1d_general(prec, direction, n, 1, 1, n * n, a, (0, 0, n * n), x, (0, 0, n * n), s)
            dfft.fft1d_strided(prec, direction, n, n, n, b, a, s)
            dfft.fft1d_contig(prec, 0, direction, n, n * n, a, n, b, n, s)
        torch.cuda.synchronize()
        assert torch.equal(out, a), f"direction {direction}: max |diff| {float((out - a).abs().max())}"
        del out, a, b
    plan.destroy()
    del x
    torch.cuda.empty_cache()
