"""Kept (untransformed) axes on one GPU: one-rank plans of every decomposition for every mask, f64 and f32, power-of-two,
Bluestein and odd shapes, against numpy over the transformed axes, with round trips, the input left intact and a canary
after `out`; R2C with y and / or x kept and mixed R2R with x kept; bit-for-bit comparisons of the x-kept output with the
full plan's d = 2 exec, in place with out of place, scaled with unscaled times s, and graph replay with eager execs; a
channel Poisson solve on a stretched wall-normal grid (tridiagonal solves along the kept x); the C++ shim; and
DFFT_ERR_STATE from the setter after an exec."""
import itertools
import os
import subprocess

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
from distributedfft_b200._lib import DfftError
from oracle import dft_oracle as O
from common import CDT, PNAME, RDT, TOL, host
from test_r2r_mixed import r2r_1d

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
MASKS = list(itertools.product((False, True), repeat=3))
KIND = {"dct": dfft.DCT, "dst": dfft.DST, "r2hc": dfft.R2HC}


def make(decomp, prec, transform, shape, axes=None, inplace=False):
    plan = CLASSES[decomp](dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if decomp == "pencil" else None, True, inplace=inplace, transform_axes=axes)
    return plan


def crand(shape, prec, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) - 0.5,
                         torch.rand(shape, generator=g, device="cuda", dtype=torch.float64) - 0.5).to(CDT[prec])


def rrand(shape, prec, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, generator=g, device="cuda", dtype=RDT[prec]) - 0.5


def ref_axes(axes, d=3):
    """numpy axes of the transformed stages among the first d (z, y, x order)"""
    return tuple(a for a in (2, 1, 0)[:d] if axes[a])


def canary_out(n, dtype):
    return torch.full((n + 64,), 7.0, dtype=dtype, device="cuda")


def canary_ok(buf):
    return bool((buf[-64:] == 7.0).all())


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp", ["slab", "zyx", "pencil"])
@pytest.mark.parametrize("shape", [(16, 32, 64), (12, 10, 7), (6, 100, 130)], ids=["pow2", "bluestein", "odd"])
def test_one_rank_every_mask(prec, decomp, shape):
    x = crand(shape, prec, 3)
    x0 = x.clone()
    xs = host(x).astype(np.complex128)
    for axes in MASKS:
        plan = make(decomp, prec, "c2c", shape, axes)
        assert plan.getTransformAxes() == axes
        ax = ref_axes(axes)
        out = canary_out(x.numel(), CDT[prec])
        plan.execC2C(out, x, dfft.FORWARD)
        got = out[:-64].reshape(shape)
        assert torch.equal(x, x0) and canary_ok(out), axes
        want = np.fft.fftn(xs, axes=ax) if ax else xs
        assert O.rel_l2(host(got), want) < TOL[prec], (axes, "forward")
        spec = got.clone()
        back = canary_out(x.numel(), CDT[prec])
        plan.execC2C(back, spec, dfft.INVERSE)
        assert torch.equal(spec, got) and canary_ok(back), axes
        n = float(np.prod([shape[a] for a in ax])) if ax else 1.0
        assert O.rel_l2(host(back[:-64].reshape(shape)) / n, xs) < TOL[prec], (axes, "round trip")
        if not any(axes):  # a pure transpose on one rank: exact
            assert torch.equal(got, x) and torch.equal(back[:-64].reshape(shape), x)
        plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp", ["slab", "pencil"])
def test_r2c_with_kept_axes(prec, decomp):
    shape = (16, 32, 64)
    x = rrand(shape, prec, 4)
    xs = host(x).astype(np.float64)
    for axes in ((False, True, True), (True, False, True), (False, False, True)):
        plan = make(decomp, prec, "r2c", shape, axes)
        osz = tuple(plan.getOutSize())
        out = canary_out(int(np.prod(osz)), CDT[prec])
        plan.execR2C(out, x)
        want = np.fft.rfft(xs, axis=2)
        for a in (1, 0):
            if axes[a]:
                want = np.fft.fft(want, axis=a)
        assert O.rel_l2(host(out[:-64].reshape(osz)), want) < TOL[prec] and canary_ok(out), axes
        back = torch.empty_like(x)
        plan.execC2R(back, out[:-64].reshape(osz).clone())
        n = shape[2] * (shape[1] if axes[1] else 1) * (shape[0] if axes[0] else 1)
        assert O.rel_l2(host(back) / n, xs) < TOL[prec], axes
        plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp", ["slab", "zyx", "pencil"])
def test_mixed_r2r_x_kept(prec, decomp):
    names, shape = ("dct", "r2hc", "dst"), (32, 64, 16)
    x = rrand(shape, prec, 5)
    xs = host(x).astype(np.float64)
    plan = make(decomp, prec, names, shape, (False, True, True))
    y = canary_out(x.numel(), RDT[prec])
    plan.execR2R(y, x, dfft.FORWARD)
    want = r2r_1d(r2r_1d(xs, dfft.DST, False, 2), dfft.R2HC, False, 1)
    assert O.rel_l2(host(y[:-64].reshape(shape)), want) < TOL[prec] and canary_ok(y)
    back = torch.empty_like(x)
    plan.execR2R(back, y[:-64].reshape(shape).clone(), dfft.INVERSE)
    assert O.rel_l2(host(back) / (shape[1] * 2 * shape[2]), xs) < TOL[prec]
    plan.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp", ["slab", "zyx", "pencil"])
def test_x_kept_equals_d2_of_full_plan(prec, decomp):
    """one rank: the x-kept exec runs the full plan's d = 2 steps, so the outputs are identical"""
    shape = (32, 64, 128)
    x = crand(shape, prec, 6)
    kept, full = make(decomp, prec, "c2c", shape, (False, True, True)), make(decomp, prec, "c2c", shape)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        a, b = torch.empty_like(x), torch.empty_like(x)
        kept.execC2C(a, x, direction)
        full.execC2C(b, x, direction, d=2)
        if not (decomp == "zyx" and direction == dfft.INVERSE):  # Z_Then_YX has no partial inverse of its own
            assert torch.equal(a, b), direction
    kept.destroy(); full.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp", ["slab", "zyx", "pencil"])
@pytest.mark.parametrize("axes", [(False, True, True), (True, False, True), (True, True, False), (False, False, False)])
def test_inplace_scale_and_graph(prec, decomp, axes):
    shape = (32, 64, 128)
    x = crand(shape, prec, 7)
    po, pi = make(decomp, prec, "c2c", shape, axes), make(decomp, prec, "c2c", shape, axes, inplace=True)
    s = 0.37
    for direction in (dfft.FORWARD, dfft.INVERSE):
        po.setScale(1.0, 1.0)
        plain = torch.empty_like(x)
        po.execC2C(plain, x, direction)
        # in place against out of place
        buf = canary_out(pi.getDomainSize() // x.element_size(), CDT[prec])
        buf[:x.numel()].copy_(x.reshape(-1))
        pi.execC2C(buf, buf, direction)
        assert torch.equal(buf[:x.numel()].reshape(shape), plain) and canary_ok(buf), (axes, direction)
        # scaled against unscaled times s
        po.setScale(s, s)
        scaled = torch.empty_like(x)
        po.execC2C(scaled, x, direction)
        assert torch.equal(scaled, plain * torch.tensor(s, dtype=RDT[prec], device="cuda")), (axes, direction)
    # graph replay against eager execs
    po.setScale(1.0, 1.0)
    out, back = torch.empty_like(x), torch.empty_like(x)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        po.execC2C(out, x, dfft.FORWARD, stream=st)
        po.execC2C(back, out, dfft.INVERSE, stream=st)
    st.synchronize()
    eager_out, eager_back = out.clone(), back.clone()
    out.zero_(); back.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cs = torch.cuda.current_stream()
        po.execC2C(out, x, dfft.FORWARD, stream=cs)
        po.execC2C(back, out, dfft.INVERSE, stream=cs)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager_out) and torch.equal(back, eager_back)
    po.destroy(); pi.destroy()


@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
@pytest.mark.parametrize("decomp", ["slab", "zyx", "pencil"])
@pytest.mark.parametrize("shape", [(16, 32, 64), (6, 10, 7)], ids=["pow2", "odd"])
def test_d1_z_kept_runs_the_contiguous_copy(prec, decomp, shape):
    """d = 1 with z kept: the z copy (kind 6, the CONTIG mapping) is the whole exec.  Out of place it equals the input
    times the scale, bit for bit; in place (identical views) it is skipped at scale 1 and scales the buffer otherwise.
    C2C and mixed R2R (the real element types)."""
    for transform in ("c2c", ("dct", "r2hc", "dst")):
        real = transform != "c2c"
        if real and shape[2] % 2:
            continue  # real-to-real plans take powers of two
        x = rrand(shape, prec, 12) if real else crand(shape, prec, 12)
        ex = (lambda p, o, i, direction: p.execR2R(o, i, direction, d=1)) if real else (lambda p, o, i, direction: p.execC2C(o, i, direction, d=1))
        po = make(decomp, prec, transform, shape, (True, True, False))
        pi = make(decomp, prec, transform, shape, (True, True, False), inplace=True)
        for s in (1.0, 0.37):
            po.setScale(s, s)
            pi.setScale(s, s)
            want = x * torch.tensor(s, dtype=RDT[prec], device="cuda") if s != 1.0 else x
            for direction in (dfft.FORWARD, dfft.INVERSE):
                out = canary_out(x.numel(), x.dtype)
                ex(po, out, x, direction)
                assert torch.equal(out[:-64].reshape(shape), want) and canary_ok(out), (transform, s, direction)
                buf = canary_out(pi.getDomainSize() // x.element_size(), x.dtype)
                buf[:x.numel()].copy_(x.reshape(-1))
                pi.enableTimer(True)
                ex(pi, buf, buf, direction)
                assert torch.equal(buf[:x.numel()].reshape(shape), want) and canary_ok(buf), (transform, s, direction, "in place")
                assert [l for l, _ in pi.stepTimes()] == ["z copy"]
                assert pi.lastLaunchCount() == (0 if s == 1.0 else 1), (transform, s, direction)
        po.destroy(); pi.destroy()


def test_setter_state_and_tune():
    shape = (16, 32, 64)
    plan = make("slab", dfft.F64, "c2c", shape)
    plan.setTransformAxes(False, True, True)
    x = crand(shape, dfft.F64, 8)
    y = torch.empty_like(x)
    plan.execC2C(y, x)
    with pytest.raises(DfftError) as e:
        plan.setTransformAxes(True, True, True)
    assert e.value.code == -4  # DFFT_ERR_STATE
    assert plan.getTransformAxes() == (False, True, True)
    assert "kept axis" in plan.tune(y, x)
    plan.destroy()
    r = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="r2c")
    with pytest.raises(DfftError):
        r.initFFT(dfft.GlobalSize(*shape), None, True, transform_axes=(True, True, False))


def test_step_labels_and_timer():
    shape = (16, 32, 64)
    plan = make("pencil", dfft.F64, "c2c", shape, (True, False, True))
    plan.enableTimer(True)
    x = crand(shape, dfft.F64, 9)
    y = torch.empty_like(x)
    plan.execC2C(y, x)
    labels = [l for l, ms in plan.stepTimes()]
    assert "y copy" in labels and "z pass" in labels and "x pass" in labels, labels
    plan.destroy()


@pytest.mark.parametrize("shape", [(64, 128, 128)])
def test_channel_poisson_stretched_x(shape):
    """Channel flow's pressure Poisson problem: periodic y and z (R2HC, (., r2hc, r2hc)), x wall-normal on a stretched grid
    of 64 points with homogeneous Neumann walls.  Forward with x kept, one tridiagonal solve per (ky, kz) column along x
    (torch), inverse with x kept; the residual of the discrete operator is checked to 1e-9."""
    nx, ny, nz = shape
    dt = torch.float64
    plan = make("slab", dfft.F64, ("dct", "r2hc", "r2hc"), shape, (False, True, True))
    # stretched wall-normal grid: tanh clustering of cell faces, cell centres xc, Neumann walls
    beta = 1.8
    s = torch.linspace(-1, 1, nx + 1, dtype=dt, device="cuda")
    xf = torch.tanh(beta * s) / np.tanh(beta)
    dxc = xf[1:] - xf[:-1]                     # cell widths
    xc = 0.5 * (xf[1:] + xf[:-1])
    dxf = xc[1:] - xc[:-1]                     # centre-to-centre distances (nx - 1)
    lower = torch.zeros(nx, dtype=dt, device="cuda"); upper = torch.zeros_like(lower)
    lower[1:] = 1.0 / (dxf * dxc[1:])
    upper[:-1] = 1.0 / (dxf * dxc[:-1])
    diag_x = -(lower + upper)                  # zero-flux walls: no ghost contribution
    ly, lz = 2 * np.pi, 2 * np.pi
    hy, hz = ly / ny, lz / nz
    ky = torch.arange(ny, dtype=dt, device="cuda")
    kz = torch.arange(nz, dtype=dt, device="cuda")
    lam_y = -4 * torch.sin(np.pi * torch.minimum(ky, ny - ky) / ny) ** 2 / hy ** 2
    lam_z = -4 * torch.sin(np.pi * torch.minimum(kz, nz - kz) / nz) ** 2 / hz ** 2
    f = rrand(shape, dfft.F64, 21)
    f -= (f * dxc.view(nx, 1, 1)).sum() / (dxc.sum() * ny * nz)  # compatible with the Neumann walls
    fh = torch.empty_like(f)
    plan.execR2R(fh, f, dfft.FORWARD)
    # tridiagonal systems along x, one per (ky, kz): lower u[i-1] + (diag + lam) u[i] + upper u[i+1] = fh[i]
    lam = (lam_y.view(ny, 1) + lam_z.view(1, nz)).reshape(-1)
    rhs = fh.reshape(nx, -1).clone()
    d = diag_x.view(nx, 1) + lam.view(1, -1)
    a = lower.view(nx, 1).expand_as(d)
    c = upper.view(nx, 1).expand_as(d)
    singular = lam == 0  # the (0, 0) column: pin u[0] = 0
    d = d.clone(); c = c.clone()
    d[0, singular] = 1.0; c[0, singular] = 0.0; rhs[0, singular] = 0.0
    cp = torch.empty_like(d); dp = torch.empty_like(d)
    cp[0] = c[0] / d[0]; dp[0] = rhs[0] / d[0]
    for i in range(1, nx):
        m = d[i] - a[i] * cp[i - 1]
        cp[i] = c[i] / m
        dp[i] = (rhs[i] - a[i] * dp[i - 1]) / m
    uh = torch.empty_like(d)
    uh[-1] = dp[-1]
    for i in range(nx - 2, -1, -1):
        uh[i] = dp[i] - cp[i] * uh[i + 1]
    u = torch.empty_like(f)
    plan.execR2R(u, uh.reshape(shape).contiguous(), dfft.INVERSE)
    u /= ny * nz  # HC2R round trips scale by N per axis
    # the discrete operator: second differences on the stretched x (Neumann walls) and periodic y, z
    lap = torch.zeros_like(u)
    lap[1:] += lower[1:].view(-1, 1, 1) * (u[:-1] - u[1:])
    lap[:-1] += upper[:-1].view(-1, 1, 1) * (u[1:] - u[:-1])
    lap += (torch.roll(u, 1, 1) + torch.roll(u, -1, 1) - 2 * u) / hy ** 2
    lap += (torch.roll(u, 1, 2) + torch.roll(u, -1, 2) - 2 * u) / hz ** 2
    res = float(torch.linalg.norm(lap - f) / torch.linalg.norm(f))
    assert res <= 1e-9, res
    plan.destroy()


def test_cpp_shim(tmp_path):
    """tests/cpp/transform_axes_shim_test.cpp: setTransformAxes through the shim against the C ABI plan, by memcmp"""
    exe = str(tmp_path / "transform_axes_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
                    os.path.join(HERE, "cpp", "transform_axes_shim_test.cpp"), "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64",
                    "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
