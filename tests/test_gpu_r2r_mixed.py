"""Real-to-real plans with a kind per axis on one GPU: the single-axis R2HC / HC2R call against the numpy halfcomplex
reference for every power of two 2..8192, CONTIG and TILED, odd line and column counts, in place; one-rank plans of each
decomposition against the per-axis reference, including the channel case (r2hc, r2hc, dct) at 512^3, partial d and
batches; bit-for-bit comparisons of in place with out of place, scaled with unscaled, three DCT kinds with the DFFT_DCT
plan and graph replay with eager execs; round trips, the input left intact, a canary after `out`, mismatched execs; a
mixed-boundary Poisson solve checked with the 7-point Laplacian; and the C++ shim's per-axis constructor."""
import os
import subprocess

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
from distributedfft_b200._lib import DfftError
from oracle import dft_oracle as O
from common import NPR, PNAME, RDT, TOL, dev, host
from test_r2r_mixed import global_ref, r2r_1d

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
KIND = {"dct": dfft.DCT, "dst": dfft.DST, "r2hc": dfft.R2HC}


def rand(shape, prec, seed):
    return np.random.default_rng(seed).standard_normal(shape).astype(NPR[prec])


def trand(shape, prec, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, generator=g, device="cuda", dtype=RDT[prec]) - 0.5


def make(names, prec, decomp, shape, batch=1, inplace=False):
    plan = CLASSES[decomp](dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=names)
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if decomp == "pencil" else None, True, batch=batch, inplace=inplace)
    return plan


def kinds_of(names):
    return tuple(KIND[n] for n in names)


def round_trip_factor(names, shape, d):
    f = 1.0
    for axis in (2, 1, 0)[:d]:
        f *= shape[axis] * (1 if names[axis] == "r2hc" else 2)
    return f


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("log2n", list(range(1, 14)))
def test_fft1d_r2hc(prec, log2n):
    n = 1 << log2n
    # (a, b): CONTIG with an odd line count, TILED with odd and even column counts
    for a, b in ((257 if n <= 256 else 7, 1), (3, 5), (2, 33), (1, 64)):
        x = rand((a, n, b), prec, n + b)
        xin = dev(x)
        out = torch.empty_like(xin)
        for direction in (dfft.FORWARD, dfft.INVERSE):
            dfft.fft1d_r2r(prec, dfft.R2HC, direction, n, a, b, out, xin)
            torch.cuda.synchronize()
            want = r2r_1d(x.astype(np.float64), dfft.R2HC, direction == dfft.INVERSE, 1)
            assert O.rel_l2(host(out), want) < TOL[prec], (a, b, direction)
            buf = xin.clone()
            dfft.fft1d_r2r(prec, dfft.R2HC, direction, n, a, b, buf, buf)
            torch.cuda.synchronize()
            assert torch.equal(buf, out), ("in place", a, b, direction)
        assert np.array_equal(host(xin), x)


PLANS = [("slab", ("r2hc", "r2hc", "dct"), (64, 32, 128), 3), ("slab", ("dst", "r2hc", "dct"), (64, 32, 128), 3),
         ("slab", ("r2hc", "dct", "dst"), (8, 8, 8192), 3), ("slab", ("r2hc", "r2hc", "r2hc"), (2, 2, 2), 3),
         ("slab", ("dct", "dst", "r2hc"), (32, 32, 32), 3),  # cubic: only the axis tells the kinds apart
         ("zyx", ("r2hc", "r2hc", "dct"), (64, 32, 128), 3), ("zyx", ("dct", "r2hc", "dst"), (16, 4096, 4), 3),
         ("pencil", ("dst", "r2hc", "dct"), (64, 32, 128), 3), ("pencil", ("r2hc", "dst", "r2hc"), (64, 32, 128), 1),
         ("pencil", ("r2hc", "r2hc", "dct"), (64, 32, 128), 2), ("slab", ("dct", "r2hc", "r2hc"), (32, 64, 16), 2)]


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp,names,shape,d", PLANS)
def test_one_rank_plans(prec, decomp, names, shape, d):
    plan = make(names, prec, decomp, shape)
    assert plan.getR2RKinds() == kinds_of(names)
    x = trand(shape, prec, 5)
    x0 = x.clone()
    osz = tuple(plan.getPartialSize(d))
    out = torch.full((int(np.prod(osz)) + 64,), 7.0, dtype=RDT[prec], device="cuda")
    plan.execR2R(out, x, dfft.FORWARD, d=d)
    got = out[:-64].reshape(osz)
    assert torch.equal(x, x0) and bool((out[-64:] == 7.0).all())
    kinds = kinds_of(names)
    assert O.rel_l2(host(got), global_ref(host(x).astype(np.float64), kinds, False, d)) < TOL[prec]
    back = torch.full((x.numel() + 64,), 7.0, dtype=RDT[prec], device="cuda")
    spec = got.clone()
    plan.execR2R(back, spec, dfft.INVERSE, d=d)
    assert torch.equal(spec, got) and bool((back[-64:] == 7.0).all())
    assert O.rel_l2(host(back[:-64].reshape(shape)), global_ref(host(spec).astype(np.float64), kinds, True, d)) < TOL[prec]
    # the round trip scales by N per R2HC axis and 2N per DCT / DST axis
    assert O.rel_l2(host(back[:-64]).reshape(shape) / round_trip_factor(names, shape, d), host(x)) < TOL[prec]
    plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
def test_channel_512(prec):
    """(r2hc, r2hc, dct) at 512^3: a 16^3 sub-block of the spectrum from the 1D transforms along each axis (separable),
    and a normalised round trip against the input"""
    names, shape = ("r2hc", "r2hc", "dct"), (512, 512, 512)
    plan = make(names, prec, "slab", shape)
    plan.setScale(1.0, 1.0 / round_trip_factor(names, shape, 3))
    x = trand(shape, prec, 8)
    y = torch.empty_like(x)
    plan.execR2R(y, x, dfft.FORWARD)
    xs = host(x).astype(np.float64)
    ks = [np.arange(0, s, s // 16) for s in shape]
    r = r2r_1d(xs, dfft.DCT, False, 2)[:, :, ks[2]]
    r = r2r_1d(r, dfft.R2HC, False, 1)[:, ks[1], :]
    r = r2r_1d(r, dfft.R2HC, False, 0)[ks[0], :, :]
    del xs
    assert O.rel_l2(host(y)[np.ix_(ks[0], ks[1], ks[2])], r) < TOL[prec] * 4
    back = torch.empty_like(x)
    plan.execR2R(back, y, dfft.INVERSE)
    assert O.rel_l2(host(back), host(x)) < TOL[prec] * 4
    plan.destroy()
    del x, y, back
    torch.cuda.empty_cache()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("names", [("r2hc", "r2hc", "dct"), ("dst", "r2hc", "dct")])
def test_batch_and_inplace(prec, names):
    shape = (16, 32, 64)
    x = trand((3,) + shape, prec, 3)
    p3, p1 = make(names, prec, "slab", shape, batch=3), make(names, prec, "slab", shape)
    pin = make(names, prec, "slab", shape, batch=3, inplace=True)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        out = torch.empty_like(x)
        p3.execR2R(out, x, direction)
        for f in range(3):
            one = torch.empty_like(x[f])
            p1.execR2R(one, x[f].contiguous(), direction)
            assert torch.equal(out[f], one), (direction, f)
            want = global_ref(host(x[f]).astype(np.float64), kinds_of(names), direction == dfft.INVERSE, 3)
            assert O.rel_l2(host(one), want) < TOL[prec]
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
    names = ("r2hc", "dst", "dct")
    x = trand(shape, prec, 6)
    po, pi = make(names, prec, decomp, shape), make(names, prec, decomp, shape, inplace=True)
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
def test_scale_bit_identical_and_round_trip(prec):
    names, shape = ("r2hc", "r2hc", "dct"), (32, 64, 128)
    x = trand(shape, prec, 9)
    plan = make(names, prec, "slab", shape)
    n = round_trip_factor(names, shape, 3)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        plain = torch.empty_like(x)
        plan.setScale(1.0, 1.0)
        plan.execR2R(plain, x, direction)
        for s in (1.0 / n, 0.3):
            plan.setScale(s, s)
            scaled = torch.empty_like(x)
            plan.execR2R(scaled, x, direction)
            st = torch.tensor(s, dtype=RDT[prec], device="cuda")
            assert torch.equal(scaled, plain * st), (direction, s)
    plan.setScale(1.0, 1.0 / n)
    y, back = torch.empty_like(x), torch.empty_like(x)
    plan.execR2R(y, x, dfft.FORWARD)
    plan.execR2R(back, y, dfft.INVERSE)
    assert O.rel_l2(host(back), host(x)) < TOL[prec]
    plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("name", ["dct", "dst"])
def test_uniform_kinds_match_the_dct_dst_plan(prec, name):
    shape = (64, 32, 128)
    x = trand(shape, prec, 11)
    a = make((name,) * 3, prec, "slab", shape)
    b = CLASSES["slab"](dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=name)
    b.initFFT(dfft.GlobalSize(*shape), None, True)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        ya, yb = torch.empty_like(x), torch.empty_like(x)
        a.execR2R(ya, x, direction)
        b.execR2R(yb, x, direction)
        assert torch.equal(ya, yb), direction
    a.destroy(); b.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
def test_graph_replay(prec):
    shape = (64, 32, 128)
    x = trand(shape, prec, 4)
    plan = make(("dst", "r2hc", "dct"), prec, "slab", shape)
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
    shape = (16, 32, 64)
    r = make(("r2hc", "r2hc", "dct"), dfft.F64, "slab", shape)
    x = trand(shape, dfft.F64, 1)
    y = torch.empty_like(x)
    for call in (lambda: r.execR2C(y, x), lambda: r.execC2R(y, x), lambda: r.execC2C(y, x)):
        with pytest.raises(DfftError) as e:
            call()
        assert e.value.code == -1
    c = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="c2c")
    c.initFFT(dfft.GlobalSize(*shape), None, True)
    with pytest.raises(DfftError) as e:
        c.getR2RKinds()
    assert e.value.code == -1
    with pytest.raises(ValueError):
        dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), transform=("r2hc", "r2c", "dct"))
    r.enableTimer(True)
    r.execR2R(y, x)
    steps = r.stepTimes()
    assert len(steps) == 3 and all(ms >= 0 for _, ms in steps)
    assert "sequential schedule" in r.tune(y, x)
    for p in (r, c):
        p.destroy()


@pytest.mark.parametrize("names", [("r2hc", "r2hc", "dct"), ("dst", "r2hc", "dct")])
def test_poisson_solve(names):
    """The 7-point discrete Poisson problem on a 32 x 64 x 128 grid: periodic R2HC axes, cell-centred Neumann (DCT) and
    Dirichlet (DST) walls.  Forward, divide by the eigenvalues of the second difference, inverse; the Laplacian of the
    result, with roll on periodic axes and ghost cells u[-1] = u[0] (Neumann) or -u[0] (Dirichlet), reproduces f."""
    shape = (32, 64, 128)
    plan = make(names, dfft.F64, "slab", shape)
    f = trand(shape, dfft.F64, 21)
    f -= f.mean()  # solvable with the (0, 0, 0) mode of the all-periodic / Neumann problem
    lam = torch.zeros(shape, dtype=torch.float64, device="cuda")
    for axis, (name, n) in enumerate(zip(names, shape)):
        k = torch.arange(n, dtype=torch.float64, device="cuda")
        if name == "r2hc":
            lk = -4 * torch.sin(np.pi * torch.minimum(k, n - k) / n) ** 2
        elif name == "dct":
            lk = -4 * torch.sin(np.pi * k / (2 * n)) ** 2
        else:
            lk = -4 * torch.sin(np.pi * (k + 1) / (2 * n)) ** 2
        view = [1, 1, 1]
        view[axis] = n
        lam = lam + lk.view(view)
    spec = torch.empty_like(f)
    plan.execR2R(spec, f, dfft.FORWARD)
    zero = lam == 0
    assert int(zero.sum()) == (1 if names[0] == "r2hc" else 0)
    spec = torch.where(zero, torch.zeros_like(spec), spec / torch.where(zero, torch.ones_like(lam), lam))
    u = torch.empty_like(f)
    plan.execR2R(u, spec.contiguous(), dfft.INVERSE)
    u /= round_trip_factor(names, shape, 3)
    lap = torch.zeros_like(u)
    for axis, name in enumerate(names):
        if name == "r2hc":
            lap += torch.roll(u, 1, axis) + torch.roll(u, -1, axis) - 2 * u
            continue
        sign = 1.0 if name == "dct" else -1.0
        first, last = u.narrow(axis, 0, 1), u.narrow(axis, u.shape[axis] - 1, 1)
        padded = torch.cat([sign * first, u, sign * last], dim=axis)
        n = u.shape[axis]
        lap += padded.narrow(axis, 0, n) + padded.narrow(axis, 2, n) - 2 * u
    err = float(torch.linalg.norm(lap - f) / torch.linalg.norm(f))
    assert err <= 1e-9, err
    plan.destroy()


def test_cpp_shim_per_axis_kinds(tmp_path):
    """tests/cpp/r2r_mixed_shim_test.cpp: the shim constructor with kinds and execR2R against the C ABI plan, by memcmp"""
    exe = str(tmp_path / "r2r_mixed_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
                    os.path.join(HERE, "cpp", "r2r_mixed_shim_test.cpp"), "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart",
                    "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
