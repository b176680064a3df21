"""Distributed 1D complex transforms (dfft_plan_create_1d) on one H100: one-rank plans of N = 2^6 .. 2^30 points against
torch.fft.fft (cuFFT) and, up to 2^16, a long-double FFT; explicit and default factors, round trips, input and canary,
the output scale, graph replay of _async execs, and 2-8 rank schedules replayed on one GPU with the real pass kernels."""
from __future__ import annotations

import numpy as np
import pytest

import fft1d_replay as F
import step_replay as R
import distributedfft_b200 as dfft

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BOUND = {"double": 1e-12, "float": 1e-5}
WORST = {}  # (precision, log2 N) -> worst rel-L2 against cuFFT, reported at the end


def setup_module():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    torch.cuda.set_device(0)


def teardown_module():
    if WORST:
        print("\nworst rel-L2 of 1D plans against torch.fft.fft:")
        for (prec, L), e in sorted(WORST.items()):
            print(f"  {prec:6s} N = 2^{L:2d}: {e:.2e}")


def make(n, precision="double", factors=None):
    torch.cuda.empty_cache()  # blocks cached by earlier sizes: a 2^30-point f64 plan needs 32 GiB of work area from the driver
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(0, 1, None, 0), precision=precision, transform="c2c")
    plan.initFFT(None, signal=n, factors=factors)
    return plan


def signal(n, cdt, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, dtype=cdt, device="cuda", generator=g)


def scrambled_error(out, ref, f):
    """rel-L2 of out [N1][N2][N3] against the natural spectrum ref, one k3 plane at a time (no full-size temporaries)"""
    n1, n2, n3 = f
    num = den = 0.0
    for k3 in range(n3):
        want = ref[n1 * n2 * k3:n1 * n2 * (k3 + 1)].view(n2, n1).t()
        num += float(torch.linalg.vector_norm((out[:, :, k3] - want).to(torch.complex128)) ** 2)
        den += float(torch.linalg.vector_norm(want.to(torch.complex128)) ** 2)
    return (num / den) ** 0.5


def ld_fft(x):
    """the DFT of x in long double (radix-2, twiddles from exact integer angles)"""
    x = np.asarray(x, dtype=np.clongdouble)
    N = x.size
    X = x.reshape(1, N)
    two_pi = np.longdouble("6.28318530717958647692528676655900577")
    while X.shape[0] < N:
        h = X.shape[1] // 2
        even, odd = X[:, :h], X[:, h:]
        a = -two_pi * np.arange(X.shape[0], dtype=np.longdouble) / np.longdouble(2 * X.shape[0])
        w = (np.cos(a) + 1j * np.sin(a)).astype(np.clongdouble)[:, None]
        X = np.vstack([even + w * odd, even - w * odd])
    return X.ravel()


@pytest.mark.parametrize("precision", ["double", "float"])
@pytest.mark.parametrize("L", range(6, 31))
def test_one_rank_against_cufft(precision, L):
    n = 1 << L
    cdt = torch.complex128 if precision == "double" else torch.complex64
    plan = make(n, precision)
    f = tuple(plan.getFactors())
    assert f[0] * f[1] * f[2] == n and tuple(plan.getInSize()) == f and tuple(plan.getOutSize()) == f
    try:
        x = signal(n, cdt, L)
        out = torch.empty(f, dtype=cdt, device="cuda")
        plan.execC2C(out, x.view(f), dfft.FORWARD)
    finally:
        plan.destroy()  # its work area, before cuFFT needs room for 2^30 points
    ref = torch.fft.fft(x)
    err = scrambled_error(out, ref, f)
    WORST[(precision, L)] = err
    assert err < BOUND[precision], err
    if L <= 16:
        want = F.scrambled(ld_fft(x.cpu().numpy()), f)
        err_ld = float(np.linalg.norm((out.cpu().numpy() - want).astype(np.complex128)) / np.linalg.norm(want.astype(np.complex128)))
        assert err_ld < BOUND[precision], err_ld


@pytest.mark.parametrize("precision", ["double", "float"])
@pytest.mark.parametrize("factors", [(8, 64, 32), (2, 2, 4096), (4096, 2, 2), (2, 8192, 2), (256, 256, 256)])
def test_explicit_factors_and_round_trip(precision, factors):
    n = int(np.prod(factors))
    cdt = torch.complex128 if precision == "double" else torch.complex64
    plan = make(n, precision, factors)
    assert tuple(plan.getFactors()) == factors
    x = signal(n, cdt, 3).view(factors)
    x_host = x.clone()
    out = torch.empty(n + 64, dtype=cdt, device="cuda")
    out[n:] = 7.5 - 2.5j  # canary after the output
    y = out[:n].view(factors)
    plan.execC2C(y, x, dfft.FORWARD)
    assert torch.equal(x, x_host), "the input changed"
    assert bool((out[n:] == 7.5 - 2.5j).all()), "a store landed after the output"
    err = scrambled_error(y, torch.fft.fft(x.reshape(-1)), factors)
    assert err < BOUND[precision], err
    back = torch.empty_like(x)
    y_host = y.clone()
    plan.execC2C(back, y, dfft.INVERSE)
    assert torch.equal(y, y_host), "the inverse's input changed"
    err = float(torch.linalg.vector_norm(back - n * x) / torch.linalg.vector_norm(n * x))
    assert err < BOUND[precision], err
    plan.destroy()


@pytest.mark.parametrize("precision", ["double", "float"])
def test_scale_is_exact(precision):
    n = 1 << 20
    cdt = torch.complex128 if precision == "double" else torch.complex64
    plan = make(n, precision)
    f = tuple(plan.getFactors())
    x = signal(n, cdt, 4).view(f)
    y1 = torch.empty_like(x)
    plan.execC2C(y1, x, dfft.FORWARD)
    b1 = torch.empty_like(x)
    plan.execC2C(b1, y1, dfft.INVERSE)
    s_f, s_i = 0.3, 1.0 / n
    plan.setScale(s_f, s_i)
    ys = torch.empty_like(x)
    plan.execC2C(ys, x, dfft.FORWARD)
    rs = torch.tensor(s_f, dtype=y1.real.dtype, device="cuda")
    assert torch.equal(torch.view_as_real(ys), torch.view_as_real(y1) * rs), "forward scale is not the unscaled output times s"
    bs = torch.empty_like(x)
    plan.execC2C(bs, y1, dfft.INVERSE)
    ri = torch.tensor(s_i, dtype=y1.real.dtype, device="cuda")
    assert torch.equal(torch.view_as_real(bs), torch.view_as_real(b1) * ri), "inverse scale is not the unscaled output times s"
    plan.destroy()


def test_graph_replay_and_tune_report():
    n = 1 << 18
    plan = make(n)
    f = tuple(plan.getFactors())
    x = signal(n, torch.complex128, 5).view(f)
    want = torch.empty_like(x)
    plan.execC2C(want, x, dfft.FORWARD)
    out = torch.empty_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        plan.execC2C(out, x, dfft.FORWARD, stream=s)  # the eager exec before capture
        g = torch.cuda.CUDAGraph()
        out.zero_()
        with torch.cuda.graph(g, stream=s):
            plan.execC2C(out, x, dfft.FORWARD, stream=s)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    x.copy_(signal(n, torch.complex128, 6).view(f))
    g.replay()
    plan.execC2C(want, x, dfft.FORWARD)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    assert "1D plans" in plan.tune(out, x, dfft.FORWARD, reps=1)
    plan.destroy()


@pytest.mark.parametrize("P, shape", [(2, (8, 8, 16)), (3, (8, 8, 8)), (4, (16, 8, 32)), (5, (8, 8, 16)), (6, (8, 16, 64)), (8, (16, 8, 32))])
@pytest.mark.parametrize("comm", [0, 1])
@pytest.mark.parametrize("inverse", [0, 1])
def test_multi_rank_replay_on_one_gpu(P, shape, comm, inverse):
    n = int(np.prod(shape))
    p = F.plan_of(P, n, shape, comm=comm)
    g = np.random.default_rng(P)
    x = g.standard_normal(shape) + 1j * g.standard_normal(shape)
    got = F.gpu_output(p, n, inverse, x)[0]
    err = R.O.rel_l2(got, F.reference(x, inverse))
    assert err < 1e-12, err
