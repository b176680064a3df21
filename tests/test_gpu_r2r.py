"""DCT / DST (real-to-real) transforms on one GPU: the single-axis call against scipy for every power of two 2..8192, CONTIG
and TILED, odd line and column counts, in place; one-rank plans of each decomposition against scipy.fft.dctn / dstn,
partial d and batches; in place against out of place and scaled against unscaled bit for bit, normalised round trips, the
input left intact, a canary after `out`, graph replay, mismatched execs, and the C++ shim's execR2R."""
import os
import subprocess

import numpy as np
import pytest
import scipy.fft as sf
import torch

import distributedfft_b200 as dfft
from distributedfft_b200._lib import DfftError
from oracle import dft_oracle as O
from common import NPR, PNAME, RDT, TOL, dev, host

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
KINDS = {dfft.DCT: "dct", dfft.DST: "dst"}


def ref1(x, kind, direction, axis):
    f = sf.dct if kind == dfft.DCT else sf.dst
    return f(x.astype(np.float64), type=2 if direction == dfft.FORWARD else 3, axis=axis)


def refn(x, kind, direction, axes):
    f = sf.dctn if kind == dfft.DCT else sf.dstn
    return f(x.astype(np.float64), type=2 if direction == dfft.FORWARD else 3, axes=axes)


def rand(shape, prec, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(NPR[prec])


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("kind", [dfft.DCT, dfft.DST])
@pytest.mark.parametrize("log2n", list(range(1, 14)))
def test_fft1d_r2r(prec, kind, log2n):
    n = 1 << log2n
    # (a, b): CONTIG with an odd line count, TILED with odd and even column counts
    for a, b in ((257 if n <= 256 else 7, 1), (3, 5), (2, 33), (1, 64)):
        x = rand((a, n, b), prec, n + b)
        xin = dev(x)
        out = torch.empty_like(xin)
        for direction in (dfft.FORWARD, dfft.INVERSE):
            dfft.fft1d_r2r(prec, kind, direction, n, a, b, out, xin)
            torch.cuda.synchronize()
            assert O.rel_l2(host(out), ref1(x, kind, direction, 1)) < TOL[prec], (a, b, direction)
            buf = xin.clone()
            dfft.fft1d_r2r(prec, kind, direction, n, a, b, buf, buf)
            torch.cuda.synchronize()
            assert torch.equal(buf, out), ("in place", a, b, direction)
        assert np.array_equal(host(xin), x)


def test_fft1d_r2r_rejects():
    x = torch.zeros(64, dtype=torch.float64, device="cuda")
    with pytest.raises(DfftError) as e:
        dfft.fft1d_r2r(dfft.F64, dfft.DCT, dfft.FORWARD, 12, 1, 1, x, x)
    assert e.value.code == -5
    with pytest.raises(DfftError) as e:
        dfft.fft1d_r2r(dfft.F64, dfft.C2C, dfft.FORWARD, 16, 1, 1, x, x)
    assert e.value.code == -1


def make(kind, prec, decomp, shape, batch=1, inplace=False):
    plan = CLASSES[decomp](dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=KINDS[kind])
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if decomp == "pencil" else None, True, batch=batch, inplace=inplace)
    return plan


def trand(shape, prec, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, generator=g, device="cuda", dtype=RDT[prec]) - 0.5


PLANS = [("slab", (64, 32, 128), 3), ("slab", (8, 8, 8192), 3), ("slab", (2, 2, 2), 3), ("zyx", (64, 32, 128), 3), ("zyx", (16, 4096, 4), 3),
         ("pencil", (64, 32, 128), 3), ("pencil", (64, 32, 128), 1), ("pencil", (64, 32, 128), 2), ("slab", (32, 64, 16), 2)]


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("kind", [dfft.DCT, dfft.DST])
@pytest.mark.parametrize("decomp,shape,d", PLANS)
def test_one_rank_plans(prec, kind, decomp, shape, d):
    plan = make(kind, prec, decomp, shape)
    x = trand(shape, prec, 5)
    x0 = x.clone()
    osz = tuple(plan.getPartialSize(d))
    assert plan.getDomainSize() == int(np.prod(shape)) * (8 if prec == dfft.F64 else 4)
    out = torch.full((int(np.prod(osz)) + 64,), 7.0, dtype=RDT[prec], device="cuda")
    plan.execR2R(out, x, dfft.FORWARD, d=d)
    got = out[:-64].reshape(osz)
    assert torch.equal(x, x0) and bool((out[-64:] == 7.0).all())
    axes = {1: (2,), 2: (1, 2), 3: (0, 1, 2)}[d]
    assert O.rel_l2(host(got), refn(host(x), kind, dfft.FORWARD, axes)) < TOL[prec]
    back = torch.full((x.numel() + 64,), 7.0, dtype=RDT[prec], device="cuda")
    spec = got.clone()
    plan.execR2R(back, spec, dfft.INVERSE, d=d)
    assert torch.equal(spec, got) and bool((back[-64:] == 7.0).all())
    assert O.rel_l2(host(back[:-64].reshape(osz if d == 3 else shape)), refn(host(spec), kind, dfft.INVERSE, axes)) < TOL[prec]
    # the round trip scales by 2^d times the product of the transformed lengths
    n = 2.0 ** d * float(np.prod([shape[a] for a in axes]))
    assert O.rel_l2(host(back[:-64]).reshape(shape) / n, host(x)) < TOL[prec]
    plan.destroy()


@pytest.mark.parametrize("prec,shape", [(dfft.F64, (256, 256, 256)), (dfft.F32, (512, 512, 512))])
def test_large_slab(prec, shape):
    """Large grids: the forward result along one line of each axis against scipy on the gathered lines, and a normalised
    round trip against the input."""
    plan = make(dfft.DCT, prec, "slab", shape)
    N = float(np.prod(shape))
    plan.setScale(1.0, 1.0 / (8 * N))
    x = trand(shape, prec, 8)
    y = torch.empty_like(x)
    plan.execR2R(y, x, dfft.FORWARD)
    # a 16^3 sub-block of the spectrum from the 1D transforms of x along each axis (separable)
    xs = host(x).astype(np.float64)
    ks = [np.arange(0, s, s // 16) for s in shape]
    r = sf.dct(xs, type=2, axis=2)[:, :, ks[2]]
    r = sf.dct(r, type=2, axis=1)[:, ks[1], :]
    r = sf.dct(r, type=2, axis=0)[ks[0], :, :]
    got = host(y)[np.ix_(ks[0], ks[1], ks[2])]
    assert O.rel_l2(got, r) < TOL[prec] * 4
    back = torch.empty_like(x)
    plan.execR2R(back, y, dfft.INVERSE)
    assert O.rel_l2(host(back), xs) < TOL[prec] * 4
    plan.destroy()
    del x, y, back
    torch.cuda.empty_cache()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("kind", [dfft.DCT, dfft.DST])
def test_batch_and_inplace(prec, kind):
    shape = (16, 32, 64)
    x = trand((3,) + shape, prec, 3)
    p3, p1 = make(kind, prec, "slab", shape, batch=3), make(kind, prec, "slab", shape)
    pin = make(kind, prec, "slab", shape, batch=3, inplace=True)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        out = torch.empty_like(x)
        p3.execR2R(out, x, direction)
        for f in range(3):
            one = torch.empty_like(x[f])
            p1.execR2R(one, x[f].contiguous(), direction)
            assert torch.equal(out[f], one), (direction, f)
        buf = torch.full((x.numel() + 64,), 7.0, dtype=RDT[prec], device="cuda")
        buf[:-64].copy_(x.reshape(-1))
        pin.execR2R(buf, buf, direction)
        assert torch.equal(buf[:-64].reshape(x.shape), out) and bool((buf[-64:] == 7.0).all()), direction
        with pytest.raises(DfftError):
            pin.execR2R(out, x, direction)
    for p in (p3, p1, pin):
        p.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp,shape,d", [("slab", (64, 32, 128), 3), ("zyx", (32, 64, 16), 3), ("pencil", (16, 32, 64), 2)])
def test_inplace_one_rank(prec, decomp, shape, d):
    x = trand(shape, prec, 6)
    po, pi = make(dfft.DST, prec, decomp, shape), make(dfft.DST, prec, decomp, shape, inplace=True)
    spec = torch.empty(int(np.prod(po.getPartialSize(d))), dtype=RDT[prec], device="cuda")
    po.execR2R(spec, x, dfft.FORWARD, d=d)
    back = torch.empty_like(x)
    po.execR2R(back, spec, dfft.INVERSE, d=d)
    buf = torch.full((pi.getDomainSize() // x.element_size() + 64,), 7.0, dtype=RDT[prec], device="cuda")
    buf[:x.numel()].copy_(x.reshape(-1))
    pi.execR2R(buf, buf, dfft.FORWARD, d=d)
    assert torch.equal(buf[:spec.numel()], spec) and bool((buf[-64:] == 7.0).all())
    pi.execR2R(buf, buf, dfft.INVERSE, d=d)
    assert torch.equal(buf[:x.numel()], back.reshape(-1)) and bool((buf[-64:] == 7.0).all())
    po.destroy(); pi.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("kind", [dfft.DCT, dfft.DST])
def test_scale_bit_identical_and_round_trip(prec, kind):
    shape = (32, 64, 128)
    x = trand(shape, prec, 9)
    plan = make(kind, prec, "slab", shape)
    N = float(np.prod(shape))
    for direction in (dfft.FORWARD, dfft.INVERSE):
        plain = torch.empty_like(x)
        plan.setScale(1.0, 1.0)
        plan.execR2R(plain, x, direction)
        for s in (1.0 / (8 * N), 0.3):
            plan.setScale(s, s)
            scaled = torch.empty_like(x)
            plan.execR2R(scaled, x, direction)
            st = torch.tensor(s, dtype=RDT[prec], device="cuda")
            assert torch.equal(scaled, plain * st), (direction, s)
    plan.setScale(1.0, 1.0 / (8 * N))
    y, back = torch.empty_like(x), torch.empty_like(x)
    plan.execR2R(y, x, dfft.FORWARD)
    plan.execR2R(back, y, dfft.INVERSE)
    assert O.rel_l2(host(back), host(x)) < TOL[prec]
    plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
def test_graph_replay(prec):
    shape = (64, 32, 128)
    x = trand(shape, prec, 4)
    plan = make(dfft.DCT, prec, "slab", shape)
    out, back = torch.empty_like(x), torch.empty_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        plan.execR2R(out, x, dfft.FORWARD, stream=s)
        plan.execR2R(back, out, dfft.INVERSE, stream=s)
    s.synchronize()
    eager_out, eager_back = out.clone(), back.clone()
    out.zero_(); back.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cs = torch.cuda.current_stream()
        plan.execR2R(out, x, dfft.FORWARD, stream=cs)
        plan.execR2R(back, out, dfft.INVERSE, stream=cs)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager_out) and torch.equal(back, eager_back)
    plan.destroy()


def test_mismatched_execs_and_timer():
    shape = (16, 16, 16)
    r = make(dfft.DCT, dfft.F64, "slab", shape)
    x = trand(shape, dfft.F64, 1)
    y = torch.empty_like(x)
    for call in (lambda: r.execR2C(y, x), lambda: r.execC2R(y, x), lambda: r.execC2C(y, x)):
        with pytest.raises(DfftError) as e:
            call()
        assert e.value.code == -1
    c = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="c2c")
    c.initFFT(dfft.GlobalSize(*shape), None, True)
    rc = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="r2c")
    rc.initFFT(dfft.GlobalSize(*shape), None, True)
    for p in (c, rc):
        with pytest.raises(DfftError) as e:
            p.execR2R(y, x)
        assert e.value.code == -1
    r.enableTimer(True)
    r.execR2R(y, x)
    steps = r.stepTimes()
    assert len(steps) == 3 and all(ms >= 0 for _, ms in steps)
    assert "DCT / DST" in r.tune(y, x)
    for p in (r, c, rc):
        p.destroy()


def test_cpp_shim_exec_r2r(tmp_path):
    """tests/cpp/r2r_shim_test.cpp: MPIcuFFT_Slab<double> DCT and DST round trips through execR2R with setScale"""
    exe = str(tmp_path / "r2r_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include", os.path.join(HERE, "cpp", "r2r_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
