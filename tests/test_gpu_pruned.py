"""Pruned plans on one GPU: forward and inverse against numpy's fftn / rfftn of the zero-embedded field on every
decomposition, bit-for-bit scale, batch, graph replay and the m = N identity, the inverse's stores confined to the data
block, multi-rank schedules with the real kernels, and the free-space convolution the plans exist for."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_pruned import fwd_ref, inv_ref

CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
C2C_, R2C_ = dfft.C2C, dfft.R2C
SL_, ZY_, PE_ = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL


def make(kind, shape, data, spec, transform, f64=True, batch=1):
    plan = CLASSES[kind](dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if kind == "pencil" else None, True, batch=batch, spectral=spec, data=data)
    return plan


def fwd(plan, x, transform, d=3):
    import torch
    osz = plan.getPartialSize(d)
    b = x.shape[0] if x.dim() == 4 else None
    cdt = torch.complex128 if x.dtype in (torch.float64, torch.complex128) else torch.complex64
    out = torch.empty(((b,) if b else ()) + tuple(osz), dtype=cdt, device="cuda")
    if transform == "c2c":
        plan.execC2C(out, x, dfft.FORWARD, d)
    else:
        plan.execR2C(out, x, d)
    torch.cuda.synchronize()
    return out


def inv(plan, X, transform, d=3, out=None):
    import torch
    isz = plan.getInSize()
    b = X.shape[0] if X.dim() == 4 else None
    rdt = X.dtype if transform == "c2c" else (torch.float64 if X.dtype == torch.complex128 else torch.float32)
    if out is None:
        out = torch.empty(((b,) if b else ()) + tuple(isz), dtype=rdt, device="cuda")
    if transform == "c2c":
        plan.execC2C(out, X, dfft.INVERSE, d)
    else:
        plan.execC2R(out, X, d)
    torch.cuda.synchronize()
    return out


def rand(shape, transform, f64, seed):
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    dt = torch.float64 if f64 else torch.float32
    x = torch.randn(shape, generator=g, dtype=dt)
    if transform == "c2c":
        x = torch.complex(x, torch.randn(shape, generator=g, dtype=dt))
    return x.cuda()


def rel(a, b):
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


CASES = [  # shape, data, spectral
    ((32, 64, 128), (16, 32, 64), None),
    ((32, 64, 128), (17, 33, 66), (21, 43, 85)),
    ((16, 32, 64), (16, 9, 64), None),
    ((8, 16, 32), (1, 16, 2), (8, 5, 32)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("kind", ["slab", "zyx", "pencil"])
def test_against_numpy(kind, transform, f64):
    tol = 1e-10 if f64 else 1e-5
    t = C2C_ if transform == "c2c" else R2C_
    for shape, data, spec in CASES:
        spec_ = shape if spec is None else spec
        plan = make(kind, shape, data, spec, transform, f64)
        assert plan.getDataSize() == list(data) and plan.getInSize() == list(data)
        x = rand(data, transform, f64, 1)
        for d in (1, 2, 3):
            if kind == "zyx" and d == 2:
                continue  # its inverse runs every pass for d = 2 (as on ordinary plans)
            X = fwd(plan, x, transform, d)
            want = fwd_ref(x.cpu().numpy().astype(np.complex128 if transform == "c2c" else np.float64), t, shape, spec_, d)
            assert rel(X.cpu().numpy(), want) < tol, (shape, data, spec, d)
            y = inv(plan, X, transform, d)
            want_y = inv_ref(want, t, shape, data, spec_, d)
            if transform == "r2c":
                want_y = want_y.real
            assert rel(y.cpu().numpy(), want_y) < tol, (shape, data, spec, d)
        plan.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
def test_512_with_256_data(transform, f64):
    """a 512^3 transform grid with 256^3 data: the forward against numpy, inverse(forward(x)) = Ntot * x"""
    import torch
    shape, data = (512, 512, 512), (256, 256, 256)
    t = C2C_ if transform == "c2c" else R2C_
    tol = 1e-10 if f64 else 1e-5
    plan = make("slab", shape, data, None, transform, f64)
    x = rand(data, transform, f64, 2)
    X = fwd(plan, x, transform)
    want = fwd_ref(x.cpu().numpy().astype(np.complex128 if transform == "c2c" else np.float64), t, shape, shape, 3)
    assert rel(X.cpu().numpy(), want) < tol
    del want
    y = inv(plan, X, transform)
    ntot = float(np.prod(shape))
    assert rel((y / ntot).cpu().numpy(), x.cpu().numpy()) < tol
    plan.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("kind", ["slab", "zyx", "pencil"])
def test_scale_batch_graph_identity(kind, transform):
    import torch
    shape, data, spec = (32, 64, 128), (17, 33, 66), (21, 43, 85)
    for f64 in (True, False):
        plan = make(kind, shape, data, spec, transform, f64)
        x = rand(data, transform, f64, 3)
        X = fwd(plan, x, transform)
        y = inv(plan, X, transform)
        # a scale is the unscaled output times s, bit for bit
        s = 0.375 if f64 else 0.3
        plan.setScale(s, 1.0 / 3.0)
        Xs, ys = fwd(plan, x, transform), inv(plan, X, transform)
        sf = torch.tensor(s, dtype=torch.float64 if f64 else torch.float32)
        si = torch.tensor(1.0 / 3.0, dtype=torch.float64 if f64 else torch.float32)
        assert torch.equal(Xs, X * sf.item() if f64 else torch.complex(X.real * sf.cuda(), X.imag * sf.cuda()))
        if transform == "c2c":
            assert torch.equal(ys, y * si.item() if f64 else torch.complex(y.real * si.cuda(), y.imag * si.cuda()))
        else:
            assert torch.equal(ys, y * si.cuda())
        plan.setScale(1.0, 1.0)
        # graph replay equals the eager exec, both directions
        stream = torch.cuda.Stream()
        out, back = torch.empty_like(X), torch.empty_like(y)

        def both(st):
            if transform == "c2c":
                plan.execC2C(out, x, dfft.FORWARD, stream=st)
                plan.execC2C(back, X, dfft.INVERSE, stream=st)
            else:
                plan.execR2C(out, x, stream=st)
                plan.execC2R(back, X, stream=st)
        both(stream)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        out.zero_()
        back.zero_()
        with torch.cuda.graph(g, stream=stream):
            both(torch.cuda.current_stream())
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, X) and torch.equal(back, y)
        plan.destroy()
        # batch: field f equals the one-field exec
        pb = make(kind, shape, data, spec, transform, f64, batch=3)
        xs = [x, rand(data, transform, f64, 4), rand(data, transform, f64, 5)]
        Xb = fwd(pb, torch.stack(xs), transform)
        yb = inv(pb, Xb, transform)
        p1 = make(kind, shape, data, spec, transform, f64)
        for f in range(3):
            Xf = fwd(p1, xs[f], transform)
            assert torch.equal(Xb[f], Xf) and torch.equal(yb[f], inv(p1, Xf, transform)), f
        p1.destroy()
        pb.destroy()
        # data = N: the padded plan of the same spectral, and the ordinary plan when both are full, bit for bit
        xn = rand(shape, transform, f64, 6)
        for spec_, ref in ((spec, make(kind, shape, None, spec, transform, f64)), (None, make(kind, shape, None, None, transform, f64))):
            pn = make(kind, shape, shape, spec_, transform, f64)
            Xr = fwd(ref, xn, transform)
            assert torch.equal(fwd(pn, xn, transform), Xr)
            assert torch.equal(inv(pn, Xr, transform), inv(ref, Xr, transform))
            pn.destroy()
            ref.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("kind", ["slab", "zyx", "pencil"])
def test_stores_stay_in_the_block(kind, transform):
    """the inverse writes only its m-blocks (canary fields after the last one stay as they were) and the forward leaves its
    input intact"""
    import torch
    shape, data = (32, 64, 128), (16, 24, 40)
    plan = make(kind, shape, data, None, transform, True, batch=2)
    x = rand((2,) + data, transform, True, 7)
    x0 = x.clone()
    X = fwd(plan, x, transform)
    assert torch.equal(x, x0)
    buf = torch.full((4,) + data, 12345.0, dtype=x.dtype, device="cuda")
    canary = buf[2:].clone()
    X0 = X.clone()
    inv(plan, X, transform, out=buf[:2])
    assert torch.equal(X, X0)
    assert torch.equal(buf[2:], canary)
    ntot = float(np.prod(shape))
    assert rel((buf[:2] / ntot).cpu().numpy(), x.cpu().numpy()) < 1e-10
    plan.destroy()


@pytest.mark.gpu
def test_tune_has_one_candidate():
    import torch
    plan = make("slab", (16, 32, 64), (8, 16, 32), None, "c2c")
    out = torch.empty(tuple(plan.getOutSize()), dtype=torch.complex128, device="cuda")
    assert "pruned plans run the sequential schedule" in plan.tune(out, rand((8, 16, 32), "c2c", True, 9))
    plan.destroy()


# ---- the free-space convolution -------------------------------------------------------------------------------------------
def direct_sum(rho):
    """phi_i = sum_j G(i - j) rho_j with G(r) = 1/|r|, G(0) = 1, over a cube of m^3 points"""
    m = rho.shape[0]
    r = np.stack(np.meshgrid(*(np.arange(m),) * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    dist = np.sqrt(((r[:, None, :] - r[None, :, :]) ** 2).sum(-1))
    np.fill_diagonal(dist, 1.0)
    return ((1.0 / dist) @ rho.reshape(-1)).reshape(rho.shape)


def green(m, n):
    """G sampled at offsets -(m-1) .. (m-1) on each axis, wrapped into the n-point grid (zero elsewhere)"""
    off = np.arange(n)
    off = np.where(off < m, off, off - n)  # index i holds offset i (i < m) or i - n
    ok = np.abs(off) <= m - 1
    o = np.meshgrid(off, off, off, indexing="ij")
    r = np.sqrt(o[0] ** 2.0 + o[1] ** 2.0 + o[2] ** 2.0)
    r[0, 0, 0] = 1.0
    mask = ok[:, None, None] & ok[None, :, None] & ok[None, None, :]
    return np.where(mask, 1.0 / r, 0.0)


@pytest.mark.gpu
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
def test_free_space_convolution(transform):
    """inverse_pruned(FFT(G) * forward_pruned(rho)) / N^3 on the doubled grid is the direct sum over the m^3 block"""
    import torch
    m, n = 16, 32
    rho = np.random.default_rng(11).standard_normal((m, m, m))
    want = direct_sum(rho)
    G = torch.from_numpy(green(m, n)).cuda()
    whole = make("slab", (n, n, n), None, None, transform)
    pruned = make("slab", (n, n, n), (m, m, m), None, transform)
    if transform == "c2c":
        Gk = fwd(whole, G.to(torch.complex128), "c2c")
        src = torch.from_numpy(rho).to(torch.complex128).cuda()
    else:
        Gk = fwd(whole, G, "r2c")
        src = torch.from_numpy(rho).cuda()
    phi = inv(pruned, Gk * fwd(pruned, src, transform), transform) / float(n) ** 3
    got = phi.cpu().numpy()
    if transform == "c2c":
        assert np.linalg.norm(got.imag) / np.linalg.norm(want) < 1e-12
        got = got.real
    assert rel(got, want) < 1e-12
    whole.destroy()
    pruned.destroy()


# ---- multi-rank schedules on one GPU --------------------------------------------------------------------------------------
def replay_gpu(P, decomp, transform, shape, data, spec, p1, p2, comm, inverse, f64):
    """every rank's pruned steps in lock step on this GPU (gpu_replay.py: the real kernels, multi-segment views, and the
    checks it makes of every plan); returns (the global output, the numpy reference)"""
    import step_replay as R
    from gpu_replay import output

    t = C2C_ if transform == "c2c" else R2C_
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=t, prec=dfft.F64 if f64 else dfft.F32, comm=comm, batch=1, data=tuple(data),
               spectral=tuple(spec))
    rng = np.random.default_rng(P * 100 + decomp * 10 + p1)
    x = rng.standard_normal(data) if t == R2C_ else rng.standard_normal(data) + 1j * rng.standard_normal(data)
    X = fwd_ref(x, t, shape, spec, 3)
    src, want = (X, inv_ref(X, t, shape, data, spec, 3)) if inverse else (x, X)
    if t == R2C_ and inverse:
        want = want.real
    return output(p, inverse, 3, src[None])[0], want


REPLAY_GRIDS = [(P, SL_, P, 1) for P in (2, 4, 8)] + [(P, ZY_, P, 1) for P in (2, 4, 8)] + \
               [(2, PE_, 2, 1), (2, PE_, 1, 2), (4, PE_, 2, 2), (4, PE_, 1, 4), (8, PE_, 4, 2), (8, PE_, 2, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("P,decomp,p1,p2", REPLAY_GRIDS)
def test_multi_rank_replay(P, decomp, p1, p2):
    """2-8 rank schedules of every decomposition, P2P and All2All, with the real kernels: against numpy, every output element
    written, and the same bits whichever rank of a step runs first"""
    shape = (16, 32, 64)
    for data, spec in (((8, 16, 32), shape), ((9, 17, 30), (11, 21, 43))):
        for transform in ("c2c", "r2c"):
            for comm in (0, 1):
                for inverse in (0, 1):
                    for f64 in (True, False):
                        got, want = replay_gpu(P, decomp, transform, shape, data, spec, p1, p2, comm, inverse, f64)
                        assert got.shape == want.shape
                        assert rel(got.astype(np.complex128), want) < (1e-12 if f64 else 1e-5), (data, transform, comm, inverse, f64)


@pytest.mark.gpu
def test_cpp_shim_pruned(tmp_path):
    """tests/cpp/pruned_shim_test.cpp: MPIcuFFT_Slab<double>::initFFT(gs, data, spectral, partition) against the ordinary plan
    on the zero-embedded field, memcmp"""
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    exe = str(tmp_path / "pruned_shim_test")
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), "-I/usr/local/cuda/include", os.path.join(here, "cpp", "pruned_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
