"""Natural-order distributed 1D transforms (dfft_plan_create_1d_natural) on one H100: one-rank plans of N = 2^6 .. 2^30
points against torch.fft.fft (cuFFT) compared directly, with no index map, and, up to 2^16, against a long-double FFT;
agreement with the scrambled plan of dfft_plan_create_1d; round trips, the exact output scale, input and canary; graph
replay of _async execs; and 2-8 rank schedules replayed on one GPU with the real pass kernels."""
from __future__ import annotations

import numpy as np
import pytest

import fft1d_natural_replay as N
import gpu_replay as G
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
        print("\nworst rel-L2 of natural-order 1D plans against torch.fft.fft:")
        for (prec, L), e in sorted(WORST.items()):
            print(f"  {prec:6s} N = 2^{L:2d}: {e:.2e}")


def make(n, precision="double", factors=None, natural=True):
    torch.cuda.empty_cache()  # blocks cached by earlier sizes: a 2^30-point f64 plan needs 32 GiB of work area from the driver
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(0, 1, None, 0), precision=precision, transform="c2c")
    plan.initFFT(None, signal=n, factors=factors, natural=natural)
    return plan


def signal(n, cdt, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(n, dtype=cdt, device="cuda", generator=g)


def rel_err(got, want, chunk=1 << 26):
    """rel-L2 of two flat tensors, a chunk at a time (no full-size temporaries at 2^30 points)"""
    num = den = 0.0
    for i in range(0, want.numel(), chunk):
        w = want[i:i + chunk].to(torch.complex128)
        num += float(torch.linalg.vector_norm(got[i:i + chunk].to(torch.complex128) - w) ** 2)
        den += float(torch.linalg.vector_norm(w) ** 2)
    return (num / den) ** 0.5


def ld_fft(x):
    """the DFT of x in long double (radix-2, twiddles from exact integer angles)"""
    x = np.asarray(x, dtype=np.clongdouble)
    n = x.size
    X = x.reshape(1, n)
    two_pi = np.longdouble("6.28318530717958647692528676655900577")
    while X.shape[0] < n:
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
    n1, n2, n3 = f = tuple(plan.getFactors())
    assert n1 * n2 * n3 == n and tuple(plan.getInSize()) == f and tuple(plan.getOutSize()) == (n3, n2, n1)
    assert tuple(plan.getOutStart()) == (0, 0, 0)
    try:
        x = signal(n, cdt, L)
        out = torch.empty((n3, n2, n1), dtype=cdt, device="cuda")
        plan.execC2C(out, x.view(f), dfft.FORWARD)
    finally:
        plan.destroy()  # its work area, before cuFFT needs room for 2^30 points
    ref = torch.fft.fft(x)
    err = rel_err(out.view(-1), ref)  # natural order: out flattened is the spectrum
    WORST[(precision, L)] = err
    assert err < BOUND[precision], err
    if L <= 16:
        want = ld_fft(x.cpu().numpy())
        got = out.view(-1).cpu().numpy()
        err_ld = float(np.linalg.norm((got - want).astype(np.complex128)) / np.linalg.norm(want.astype(np.complex128)))
        assert err_ld < BOUND[precision], err_ld


@pytest.mark.parametrize("precision", ["double", "float"])
@pytest.mark.parametrize("L", [10, 16, 20, 24])
def test_agrees_with_scrambled_plan(precision, L):
    """On one rank the natural plan runs the scrambled plan's x and y passes and the same core, stage plan and tables in
    its transposing z pass: its output is the scrambled output, index-mapped, bit for bit."""
    n = 1 << L
    cdt = torch.complex128 if precision == "double" else torch.complex64
    x = signal(n, cdt, 100 + L)
    nat, scr = make(n, precision), make(n, precision, natural=False)
    f = tuple(scr.getFactors())
    assert tuple(nat.getFactors()) == f
    a = torch.empty(f[::-1], dtype=cdt, device="cuda")
    b = torch.empty(f, dtype=cdt, device="cuda")
    nat.execC2C(a, x.view(f), dfft.FORWARD)
    scr.execC2C(b, x.view(f), dfft.FORWARD)
    assert torch.equal(a, b.permute(2, 1, 0)), rel_err(a.reshape(-1), b.permute(2, 1, 0).reshape(-1))
    # and the inverses of the same spectrum
    ia, ib = torch.empty_like(b), torch.empty_like(b)
    nat.execC2C(ia, a, dfft.INVERSE)
    scr.execC2C(ib, b, dfft.INVERSE)
    assert torch.equal(ia, ib), rel_err(ia.reshape(-1), ib.reshape(-1))
    nat.destroy()
    scr.destroy()


@pytest.mark.parametrize("precision", ["double", "float"])
@pytest.mark.parametrize("factors", [(8, 64, 32), (2, 2, 4096), (4096, 2, 2), (2, 8192, 2), (256, 256, 256), (1024, 64, 16)])
def test_explicit_factors_and_round_trip(precision, factors):
    n = int(np.prod(factors))
    cdt = torch.complex128 if precision == "double" else torch.complex64
    plan = make(n, precision, factors)
    assert tuple(plan.getFactors()) == factors
    x = signal(n, cdt, 3).view(factors)
    x_host = x.clone()
    out = torch.empty(n + 64, dtype=cdt, device="cuda")
    out[n:] = 7.5 - 2.5j  # canary after the output
    y = out[:n].view(factors[::-1])
    plan.execC2C(y, x, dfft.FORWARD)
    assert torch.equal(x, x_host), "the input changed"
    assert bool((out[n:] == 7.5 - 2.5j).all()), "a store landed after the output"
    err = rel_err(y.reshape(-1), torch.fft.fft(x.reshape(-1)))
    assert err < BOUND[precision], err
    back = torch.empty(n + 64, dtype=cdt, device="cuda")
    back[n:] = 7.5 - 2.5j
    y_host = y.clone()
    plan.execC2C(back[:n].view(factors), y, dfft.INVERSE)
    assert torch.equal(y, y_host), "the inverse's input changed"
    assert bool((back[n:] == 7.5 - 2.5j).all()), "a store landed after the inverse's output"
    err = rel_err(back[:n], n * x.reshape(-1))
    assert err < BOUND[precision], err
    plan.destroy()


@pytest.mark.parametrize("precision", ["double", "float"])
def test_scale_is_exact(precision):
    n = 1 << 20
    cdt = torch.complex128 if precision == "double" else torch.complex64
    plan = make(n, precision)
    f = tuple(plan.getFactors())
    x = signal(n, cdt, 4).view(f)
    y1 = torch.empty(f[::-1], dtype=cdt, device="cuda")
    plan.execC2C(y1, x, dfft.FORWARD)
    b1 = torch.empty_like(x)
    plan.execC2C(b1, y1, dfft.INVERSE)
    s_f, s_i = 0.3, 1.0 / n
    plan.setScale(s_f, s_i)
    ys = torch.empty_like(y1)
    plan.execC2C(ys, x, dfft.FORWARD)
    rs = torch.tensor(s_f, dtype=y1.real.dtype, device="cuda")
    assert torch.equal(torch.view_as_real(ys), torch.view_as_real(y1) * rs), "forward scale is not the unscaled output times s"
    bs = torch.empty_like(x)
    plan.execC2C(bs, y1, dfft.INVERSE)
    ri = torch.tensor(s_i, dtype=y1.real.dtype, device="cuda")
    assert torch.equal(torch.view_as_real(bs), torch.view_as_real(b1) * ri), "inverse scale is not the unscaled output times s"
    assert rel_err(bs.reshape(-1), x.reshape(-1)) < BOUND[precision]
    plan.destroy()


def test_graph_replay_and_tune_report():
    n = 1 << 18
    plan = make(n)
    f = tuple(plan.getFactors())
    x = signal(n, torch.complex128, 5).view(f)
    want = torch.empty(f[::-1], dtype=torch.complex128, device="cuda")
    plan.execC2C(want, x, dfft.FORWARD)
    out = torch.empty_like(want)
    back = torch.empty_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        plan.execC2C(out, x, dfft.FORWARD, stream=s)  # the eager execs before capture
        plan.execC2C(back, out, dfft.INVERSE, stream=s)
        g = torch.cuda.CUDAGraph()
        out.zero_()
        with torch.cuda.graph(g, stream=s):
            plan.execC2C(out, x, dfft.FORWARD, stream=s)
            plan.execC2C(back, out, dfft.INVERSE, stream=s)
    out.zero_()
    back.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    assert rel_err(back.reshape(-1), n * x.reshape(-1)) < BOUND["double"]
    x.copy_(signal(n, torch.complex128, 6).view(f))
    g.replay()
    plan.execC2C(want, x, dfft.FORWARD)
    torch.cuda.synchronize()
    assert torch.equal(out, want)
    assert "1D plans" in plan.tune(out, x, dfft.FORWARD, reps=1)
    plan.destroy()


@pytest.mark.parametrize("P, shape", [(2, (8, 8, 16)), (3, (8, 8, 8)), (4, (16, 8, 32)), (5, (8, 8, 16)), (6, (8, 16, 64)),
                                      (7, (16, 8, 8)), (8, (16, 8, 32)), (3, (64, 32, 1024))])
@pytest.mark.parametrize("comm", [0, 1])
@pytest.mark.parametrize("inverse", [0, 1])
def test_multi_rank_replay_on_one_gpu(P, shape, comm, inverse):
    n = int(np.prod(shape))
    p = N.plan_of(P, n, shape, comm=comm)
    g = np.random.default_rng(P)
    x = g.standard_normal(shape[::-1] if inverse else shape) + 1j * g.standard_normal(shape[::-1] if inverse else shape)
    got = N.gpu_output(p, n, inverse, x)
    err = R.O.rel_l2(got, N.reference(x, inverse))
    assert err < 1e-12, err
    again = N.gpu_output(p, n, inverse, x, descending=True)
    assert G.same_bits(again, got), "the result depends on the order of the ranks within a step"


@pytest.mark.parametrize("comm", [0, 1])
@pytest.mark.parametrize("inverse", [0, 1])
def test_multi_rank_replay_scale(comm, inverse):
    """With an output scale on three ranks, the step that stores into the caller's out (the landing copy forward, the copy
    back to the x-slabs inverse) scales each value once: a power-of-two scale gives the unscaled output times s exactly."""
    P, shape = 3, (8, 8, 16)
    n = int(np.prod(shape))
    s = (0.5, 0.25)
    g = np.random.default_rng(11)
    x = g.standard_normal(shape[::-1] if inverse else shape) + 1j * g.standard_normal(shape[::-1] if inverse else shape)
    plain = N.gpu_output(N.plan_of(P, n, shape, comm=comm), n, inverse, x)
    got = N.gpu_output(N.plan_of(P, n, shape, comm=comm, scale=s), n, inverse, x)
    assert np.array_equal(got, plain * s[inverse])
    assert R.O.rel_l2(got, s[inverse] * N.reference(x, inverse)) < 1e-12


def test_row_side_extent_is_checked():
    """dfft_debug_run_step measures the row side of the transposing z pass with its line stride sB: a work area one element
    short of that extent is refused before anything runs, the exact extent is enough"""
    shape = (8, 16, 32)
    n = int(np.prod(shape))
    p = N.plan_of(1, n, shape)
    with N.dry_plans(p, n) as (plan,):
        sc = R.schedule(p, plan, 0, 3)
        es = sc["esize"]
        k = [i for i, st in enumerate(sc["steps"]) if st.get("label") == "z pass"][0]
        st = sc["steps"][k]
        seg = st["in"]["segs"][0]  # forward: the row side, my x-slab in the work area
        need = G.work_offset(seg["base"]) + ((st["B"] - 1) * st["transposed"] + (st["A0"] - 1) * seg["sA0"] + shape[2]) * es
        work_bytes = sc["nslots"] * sc["slot_bytes"]
        assert need <= work_bytes
        _, _, bi, bo, _ = G.caller_buffers(p, sc, 0, 3, np.zeros((1,) + shape))
        work = [G.nan_buffer(work_bytes)]
        torch.cuda.synchronize()
        before = bo.clone()
        assert G.run_step(plan, 0, 3, 0, k, work, need - es, bo, bo.numel(), bi, bi.numel()) == -1
        torch.cuda.synchronize()
        assert torch.equal(bo, before), "a refused step wrote"
        assert G.run_step(plan, 0, 3, 0, k, work, need, bo, bo.numel(), bi, bi.numel()) == 0
        torch.cuda.synchronize()
