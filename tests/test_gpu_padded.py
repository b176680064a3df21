"""Padded plans on one GPU: forward and inverse against numpy's fftn / rfftn through the index map on every decomposition,
round trips, bit-for-bit scale, batch, graph replay and K = N identity, and the dealiasing property the plans exist for."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
from test_padded import fwd_ref, inv_ref

CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
C2C_, R2C_ = dfft.C2C, dfft.R2C
SL_, ZY_, PE_ = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL


def make(kind, shape, spec, transform, f64=True, batch=1):
    plan = CLASSES[kind](dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if kind == "pencil" else None, True, batch=batch,
                 spectral=None if spec is None else spec)
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


def inv(plan, X, transform, d=3):
    import torch
    isz = plan.getInSize()
    b = X.shape[0] if X.dim() == 4 else None
    if transform == "c2c":
        out = torch.empty(((b,) if b else ()) + tuple(isz), dtype=X.dtype, device="cuda")
        plan.execC2C(out, X, dfft.INVERSE, d)
    else:
        rdt = torch.float64 if X.dtype == torch.complex128 else torch.float32
        out = torch.empty(((b,) if b else ()) + tuple(isz), dtype=rdt, device="cuda")
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


CASES = [  # shape, spec
    ((32, 64, 128), (21, 43, 85)),
    ((16, 32, 64), (16, 21, 42)),
    ((8, 16, 32), (1, 16, 21)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("kind", ["slab", "zyx", "pencil"])
def test_against_numpy(kind, transform, f64):
    tol = 1e-10 if f64 else 1e-5
    t = C2C_ if transform == "c2c" else R2C_
    for shape, spec in CASES:
        plan = make(kind, shape, spec, transform, f64)
        assert plan.getSpectralSize() == list(spec)
        x = rand(shape, transform, f64, 1)
        for d in (1, 2, 3):
            if kind == "zyx" and d == 2:
                continue  # its inverse runs every pass for d = 2 (as on ordinary plans)
            X = fwd(plan, x, transform, d)
            want = fwd_ref(x.cpu().numpy().astype(np.complex128 if transform == "c2c" else np.float64), t, spec, d)
            assert rel(X.cpu().numpy(), want) < tol, (shape, spec, d)
            y = inv(plan, X, transform, d)
            want_y = inv_ref(want, t, shape, spec, d)
            if transform == "r2c":
                want_y = want_y.real
            assert rel(y.cpu().numpy(), want_y) < tol, (shape, spec, d)
        plan.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
def test_512_two_thirds(transform, f64):
    """512^3 with K = 341 (|k| <= 170, the 2/3 rule): forward against numpy, forward(inverse(X)) = Ntot * X"""
    import torch
    shape, spec = (512, 512, 512), (341, 341, 341)
    t = C2C_ if transform == "c2c" else R2C_
    plan = make("slab", shape, spec, transform, f64)
    x = rand(shape, transform, f64, 2)
    X = fwd(plan, x, transform)
    # numpy on the whole grid (complex128)
    want = fwd_ref(x.cpu().numpy().astype(np.complex128 if transform == "c2c" else np.float64), t, spec, 3)
    assert rel(X.cpu().numpy(), want) < (1e-10 if f64 else 1e-5)
    del want
    Y = fwd(plan, inv(plan, X, transform), transform)
    ntot = float(np.prod(shape))
    assert rel((Y / ntot).cpu().numpy(), X.cpu().numpy()) < (1e-10 if f64 else 1e-5)
    plan.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("kind", ["slab", "zyx", "pencil"])
def test_scale_batch_graph_identity(kind, transform):
    import torch
    shape, spec = (32, 64, 128), (21, 43, 85)
    for f64 in (True, False):
        plan = make(kind, shape, spec, transform, f64)
        x = rand(shape, transform, f64, 3)
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
        # graph replay equals the eager exec
        stream = torch.cuda.Stream()
        out = torch.empty_like(X)
        if transform == "c2c":
            plan.execC2C(out, x, dfft.FORWARD, stream=stream)
        else:
            plan.execR2C(out, x, stream=stream)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        out.zero_()
        with torch.cuda.graph(g, stream=stream):
            if transform == "c2c":
                plan.execC2C(out, x, dfft.FORWARD, stream=torch.cuda.current_stream())
            else:
                plan.execR2C(out, x, stream=torch.cuda.current_stream())
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, X)
        plan.destroy()
        # batch equals the per-field output
        pb = make(kind, shape, spec, transform, f64, batch=3)
        xb = torch.stack([x, rand(shape, transform, f64, 4), rand(shape, transform, f64, 5)])
        Xb = fwd(pb, xb, transform)
        assert torch.equal(Xb[0], X)
        yb = inv(pb, Xb, transform)
        assert torch.equal(yb[0], y)
        pb.destroy()
        # a K = N padded plan is the ordinary plan
        pa, pn = make(kind, shape, shape, transform, f64), make(kind, shape, None, transform, f64)
        assert torch.equal(fwd(pa, x, transform), fwd(pn, x, transform))
        Xn = fwd(pn, x, transform)
        assert torch.equal(inv(pa, Xn, transform), inv(pn, Xn, transform))
        pa.destroy()
        pn.destroy()


def alias_free_product(U, V, K):
    """the exact convolution of two K^3 spectra (numpy fftfreq order), restricted to the K grid, on a 2K grid"""
    M = 2 * K
    pos = np.fft.fftfreq(K, 1.0 / K).astype(np.int64) % M
    Ue = np.zeros((M, M, M), dtype=np.complex128)
    Ve = np.zeros((M, M, M), dtype=np.complex128)
    Ue[np.ix_(pos, pos, pos)] = U
    Ve[np.ix_(pos, pos, pos)] = V
    W = np.fft.fftn(np.fft.ifftn(Ue) * np.fft.ifftn(Ve)) * M ** 3
    return W[np.ix_(pos, pos, pos)]


@pytest.mark.gpu
def test_dealiasing():
    """forward(inverse(U) * inverse(V)) / Ntot on a 3/2 grid is the alias-free convolution; on the K grid it is not"""
    import torch
    K = 21
    N = 32  # >= (3K - 1) / 2
    rng = np.random.default_rng(7)
    U = rng.standard_normal((K,) * 3) + 1j * rng.standard_normal((K,) * 3)
    V = rng.standard_normal((K,) * 3) + 1j * rng.standard_normal((K,) * 3)
    want = alias_free_product(U, V, K)

    def product(plan, n):
        u = inv(plan, torch.from_numpy(U).cuda(), "c2c")
        v = inv(plan, torch.from_numpy(V).cuda(), "c2c")
        return (fwd(plan, u * v, "c2c") / float(n) ** 3).cpu().numpy()

    padded = make("slab", (N, N, N), (K, K, K), "c2c")
    got = product(padded, N)
    padded.destroy()
    # the inverse gives sum_p U_p e^{+i p x}; the product's forward / N^3 is the convolution sum_{p+q=k} U_p V_q modulo N,
    # free of aliases on the K grid when N >= (3K - 1) / 2
    assert rel(got, want) < 1e-12
    plain = make("slab", (K, K, K), None, "c2c")
    assert rel(product(plain, K), want) > 1e-3
    plain.destroy()


# ---- multi-rank schedules on one GPU --------------------------------------------------------------------------------------
def replay_gpu(P, decomp, transform, shape, spec, p1, p2, comm, inverse, f64):
    """every rank's padded steps in lock step on this GPU (gpu_replay.py: the real kernels, multi-segment views, and the
    checks it makes of every plan); returns (the global output, the numpy reference)"""
    import step_replay as R
    from gpu_replay import output

    t = C2C_ if transform == "c2c" else R2C_
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=t, prec=dfft.F64 if f64 else dfft.F32, comm=comm, batch=1, spectral=tuple(spec))
    rng = np.random.default_rng(P * 100 + decomp * 10 + p1)
    x = rng.standard_normal(shape) if t == R2C_ else rng.standard_normal(shape) + 1j * rng.standard_normal(shape)
    X = fwd_ref(x, t, spec, 3)
    src, want = (X, inv_ref(X, t, shape, spec, 3)) if inverse else (x, X)
    if t == R2C_ and inverse:
        want = want.real
    return output(p, inverse, 3, src[None])[0], want


REPLAY_GRIDS = [(P, SL_, P, 1) for P in (2, 4, 8)] + [(P, ZY_, P, 1) for P in (2, 4, 8)] + \
               [(2, PE_, 2, 1), (2, PE_, 1, 2), (4, PE_, 2, 2), (4, PE_, 1, 4), (8, PE_, 4, 2), (8, PE_, 2, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("P,decomp,p1,p2", REPLAY_GRIDS)
def test_multi_rank_replay(P, decomp, p1, p2):
    """2-8 rank schedules of every decomposition, P2P and All2All, with the real padded kernels: against numpy, every output
    element written, and the same bits whichever rank of a step runs first"""
    shape, spec = (16, 32, 64), (11, 21, 43)
    for transform in ("c2c", "r2c"):
        for comm in (0, 1):
            for inverse in (0, 1):
                for f64 in (True, False):
                    got, want = replay_gpu(P, decomp, transform, shape, spec, p1, p2, comm, inverse, f64)
                    assert got.shape == want.shape
                    assert rel(got.astype(np.complex128), want) < (1e-12 if f64 else 1e-5), (transform, comm, inverse, f64)


@pytest.mark.gpu
def test_cpp_shim_padded(tmp_path):
    """tests/cpp/padded_shim_test.cpp: MPIcuFFT_Slab<double>::initFFT(gs, spectral, partition) against the ordinary plan,
    memcmp"""
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    exe = str(tmp_path / "padded_shim_test")
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), "-I/usr/local/cuda/include", os.path.join(here, "cpp", "padded_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
