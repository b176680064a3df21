"""C2C transforms of axis lengths that are not powers of two (the Bluestein pass) on one GPU: the single-axis calls against
numpy, one-rank plans against numpy and single-GPU cuFFT (oracle/cufft_ref.cu takes any size), round trips, the input
left intact, a canary after `out` untouched, batches, the output scale bit for bit, and graph replay."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
from oracle import dft_oracle as O
from common import CDT, NPC, TOL, dev, host

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}


def npfft(x, direction, axis):
    x = x.astype(np.complex128)
    return np.fft.fft(x, axis=axis) if direction == dfft.FORWARD else np.fft.ifft(x, axis=axis) * x.shape[axis]


def rand(shape, prec, seed):
    rng = np.random.default_rng(seed)
    return (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(NPC[prec])


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("n", [3, 5, 6, 7, 12, 17, 31, 96, 100, 127, 243, 384, 625, 1000, 1025, 2049, 3000, 4093, 4095])
def test_contig(prec, n):
    lines = 37 if n >= 64 else 301
    x = rand((lines, n), prec, n)
    xin = dev(x)
    out = torch.empty_like(xin)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        dfft.fft1d_contig(prec, 0, direction, n, lines, out, n, xin, n)
        torch.cuda.synchronize()
        assert O.rel_l2(host(out), npfft(x, direction, 1)) < TOL[prec]
    assert np.array_equal(host(xin), x)
    buf = xin.clone()  # in place
    dfft.fft1d_contig(prec, 0, dfft.INVERSE, n, lines, buf, n, buf, n)
    torch.cuda.synchronize()
    assert O.rel_l2(host(buf), npfft(x, dfft.INVERSE, 1)) < TOL[prec]


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("a,n,b", [(3, 5, 1), (2, 100, 1), (1, 3000, 1), (3, 7, 37), (2, 96, 33), (1, 625, 129), (2, 1000, 7), (1, 4093, 5),
                                   (2, 384, 16)])
def test_strided_and_general(prec, a, n, b):
    x = rand((a, n, b), prec, n + b)
    xin = dev(x)
    out = torch.empty_like(xin)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        dfft.fft1d_strided(prec, direction, a, n, b, out, xin)
        torch.cuda.synchronize()
        assert O.rel_l2(host(out), npfft(x, direction, 1)) < TOL[prec]
    buf = xin.clone()
    dfft.fft1d_strided(prec, dfft.FORWARD, a, n, b, buf, buf)
    torch.cuda.synchronize()
    assert O.rel_l2(host(buf), npfft(x, dfft.FORWARD, 1)) < TOL[prec]
    # general: the same lines read as (a0 = a, a1 = b, n, b = 1) with element strides, written transposed
    outg = torch.empty((b, a, n), dtype=CDT[prec], device="cuda")
    dfft.fft1d_general(prec, dfft.INVERSE, n, a, b, 1, outg, (n, a * n, 1), xin, (n * b, 1, b))
    torch.cuda.synchronize()
    assert O.rel_l2(host(outg), npfft(x, dfft.INVERSE, 1).transpose(2, 0, 1)) < TOL[prec]
    assert np.array_equal(host(xin), x)


def cufft_lib():
    path = os.path.join(ROOT, "oracle", "_ref", "libcufft_ref.so")
    lib = C.CDLL(path)
    lib.cufft_ref_3d.restype = C.c_int
    lib.cufft_ref_3d.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int]
    return lib


def gpu_rel(a, b):
    return float((a - b).abs().pow(2).sum().sqrt() / b.abs().pow(2).sum().sqrt())


PLANS = [("slab", (96, 96, 96), 3), ("slab", (100, 120, 90), 3), ("slab", (3, 5, 7), 3), ("slab", (17, 2048, 6), 3), ("slab", (384, 384, 384), 3),
         ("zyx", (100, 120, 90), 3), ("zyx", (96, 64, 7), 3), ("pencil", (100, 120, 90), 3), ("pencil", (12, 96, 100), 1),
         ("pencil", (12, 96, 100), 2)]


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("kind,shape,d", PLANS)
def test_one_rank_plans(prec, kind, shape, d):
    plan = CLASSES[kind](dfft.Configurations(), dfft.Comm(), precision="double" if prec == dfft.F64 else "float", transform="c2c")
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if kind == "pencil" else None, True)
    g = torch.Generator(device="cuda").manual_seed(11)
    rdt = torch.float64 if prec == dfft.F64 else torch.float32
    x = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
    x0 = x.clone()
    osz = tuple(plan.getPartialSize(d))
    out = torch.full((int(np.prod(osz)) + 64,), 7.0, dtype=CDT[prec], device="cuda")
    plan.execC2C(out, x, dfft.FORWARD, d=d)
    got = out[:-64].reshape(osz)
    assert torch.equal(x, x0) and bool((out[-64:] == 7.0).all())
    axes = {1: (2,), 2: (1, 2), 3: (0, 1, 2)}[d]
    if np.prod(shape) <= 2_000_000:
        assert O.rel_l2(host(got), np.fft.fftn(host(x).astype(np.complex128), axes=axes)) < TOL[prec]
    if d == 3:
        ref = torch.empty_like(x)
        ms = C.c_float()
        assert cufft_lib().cufft_ref_3d(1 if prec == dfft.F64 else 0, 0, *shape, ref.data_ptr(), x.data_ptr(), C.byref(ms), 1) == 0
        assert gpu_rel(got, ref) < TOL[prec]
        del ref
    back = torch.full((x.numel() + 64,), 7.0, dtype=CDT[prec], device="cuda")
    spec = got.clone()
    plan.execC2C(back, spec, dfft.INVERSE, d=d)
    assert torch.equal(spec, got) and bool((back[-64:] == 7.0).all())
    n = float(np.prod([shape[a] for a in axes]))
    assert gpu_rel(back[:-64].reshape(shape) / n, x) < TOL[prec]
    plan.destroy()
    del x, x0, out, back, spec
    torch.cuda.empty_cache()


def make(shape, prec, batch=1):
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if prec == dfft.F64 else "float", transform="c2c")
    plan.initFFT(dfft.GlobalSize(*shape), None, True, batch=batch)
    return plan


def crand(shape, prec, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rdt = torch.float64 if prec == dfft.F64 else torch.float32
    return torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt) - 0.5, torch.rand(shape, generator=g, device="cuda", dtype=rdt) - 0.5)


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
def test_batch_matches_single_fields(prec):
    shape = (12, 100, 130)
    x = crand((3,) + shape, prec, 3)
    p3, p1 = make(shape, prec, 3), make(shape, prec, 1)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        out = torch.empty_like(x)
        p3.execC2C(out, x, direction)
        for f in range(3):
            one = torch.empty_like(x[f])
            p1.execC2C(one, x[f].contiguous(), direction)
            assert torch.equal(out[f], one), (direction, f)
    p3.destroy(); p1.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("shape", [(96, 96, 96), (17, 2048, 6), (3, 5, 7)])
def test_scale_is_bit_identical(prec, shape):
    x = crand(shape, prec, 9)
    plan = make(shape, prec)
    N = float(np.prod(shape))
    for direction in (dfft.FORWARD, dfft.INVERSE):
        plain = torch.empty_like(x)
        plan.setScale(1.0, 1.0)
        plan.execC2C(plain, x, direction)
        for s in (1.0 / N, 0.3):
            plan.setScale(s, s)
            scaled = torch.empty_like(x)
            plan.execC2C(scaled, x, direction)
            st = torch.tensor(s, dtype=torch.float64 if prec == dfft.F64 else torch.float32, device="cuda")
            assert torch.equal(torch.view_as_real(scaled), torch.view_as_real(plain) * st), (direction, s)
    plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
def test_graph_replay(prec):
    shape = (100, 120, 90)
    x = crand(shape, prec, 4)
    plan = make(shape, prec)
    out, back = torch.empty_like(x), torch.empty_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        plan.execC2C(out, x, dfft.FORWARD, stream=s)
        plan.execC2C(back, out, dfft.INVERSE, stream=s)
    s.synchronize()
    eager_out, eager_back = out.clone(), back.clone()
    out.zero_(); back.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cs = torch.cuda.current_stream()
        plan.execC2C(out, x, dfft.FORWARD, stream=cs)
        plan.execC2C(back, out, dfft.INVERSE, stream=cs)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager_out) and torch.equal(back, eager_back)
    plan.destroy()
