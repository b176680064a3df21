"""Type-I real-to-real kinds (DCT-I / DST-I) on one GPU.

- dfft_fft1d_r2r with DFFT_DCT1 / DFFT_DST1 at every length, CONTIG and TILED, in place and out of place, against scipy's
  dct / dst(type=1); forward and inverse run the same transform.
- Per-line accuracy against long double at every length: lines of mixed magnitudes (1, 2^20, 2^-20, 0 in turn) held to the
  bounds of test_gpu_accuracy on each line's own norm, zero lines exact zeros.
- One-rank plans (slab, Z_Then_YX, pencil) against scipy's dctn / dstn(type=1) and the per-axis reference: 129^3, 257^3,
  (129, 128, 128) with (dct1, r2hc, r2hc), (127, 255, 63) DST-I, partial d; round trips scale by 2N per type-I axis; 513^3
  DCT-I compared on the device.
- Bit for bit: in place against out of place, batch against single fields, scale against unscaled, graph replay against
  eager.
- 2-8 rank schedules replayed with the real kernels through dfft_debug_run_step (gpu_replay.py).
- A vertex-centred Dirichlet Poisson solve with DST-I (7-point Laplacian residual) and the Chebyshev check: the DCT-I of
  T_m(cos(pi j / N)) is N delta_km, 2N at m = 0 and m = N.
- The C++ shim's per-axis constructor with type-I kinds (tests/cpp/r2r1_shim_test.cpp)."""
import math
import os
import subprocess

import numpy as np
import pytest
import scipy.fft as sf
import torch

import distributedfft_b200 as dfft
import step_replay as R
from common import PNAME, RDT, TOL
from oracle import dft_oracle as O
from test_gpu_accuracy import check_units, mixed, on_device, spec as acc_spec
from gpu_replay import output
from test_gpu_schedule_replay import global_input
from test_r2r1 import DCT1, DST1, R2HC, DCT, DST, axis_len, global_ref, r2r_1d

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
KIND = {"dct": DCT, "dst": DST, "r2hc": R2HC, "dct1": DCT1, "dst1": DST1}
F32, F64 = dfft.F32, dfft.F64
LENGTHS = [(DCT1, (1 << k) + 1) for k in range(1, 14)] + [(DST1, (1 << k) - 1) for k in range(2, 14)]


def lid(v):
    return f"{'dct1' if v[0] == DCT1 else 'dst1'}-{v[1]}"


def trand(shape, prec, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(shape, generator=g, device="cuda", dtype=RDT[prec]) - 0.5


def make(names, prec, decomp, shape, batch=1, inplace=False):
    plan = CLASSES[decomp](dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=names)
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if decomp == "pencil" else None, True, batch=batch, inplace=inplace)
    return plan


def kinds_of(names):
    return tuple(KIND[n] for n in names)


def round_trip_factor(names, shape, d=3):
    f = 1.0
    for axis in (2, 1, 0)[:d]:
        n, k = shape[axis], names[axis]
        f *= {"r2hc": n, "dct": 2 * n, "dst": 2 * n, "dct1": 2 * (n - 1), "dst1": 2 * (n + 1)}[k]
    return f


# ---- the single-axis call ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("kind,n", LENGTHS, ids=[lid(v) for v in LENGTHS])
def test_fft1d(prec, kind, n):
    for a, b in ((257 if n <= 257 else 7, 1), (3, 5), (2, 33), (1, 64)):  # CONTIG odd line count, TILED partial tiles
        x = np.random.default_rng(n + b).standard_normal((a, n, b)).astype(np.float64 if prec == F64 else np.float32)
        xin = torch.from_numpy(x).cuda()
        outs = []
        for direction in (dfft.FORWARD, dfft.INVERSE):
            out = torch.empty_like(xin)
            dfft.fft1d_r2r(prec, kind, direction, n, a, b, out, xin)
            torch.cuda.synchronize()
            assert O.rel_l2(out.cpu().numpy(), r2r_1d(x.astype(np.float64), kind, False, 1)) < TOL[prec], (a, b, direction)
            buf = xin.clone()
            dfft.fft1d_r2r(prec, kind, direction, n, a, b, buf, buf)
            torch.cuda.synchronize()
            assert torch.equal(buf, out), ("in place", a, b, direction)
            outs.append(out)
        assert torch.equal(outs[0], outs[1]), "forward and inverse are the same transform"
        assert np.array_equal(xin.cpu().numpy(), x)


@pytest.mark.parametrize("prec", [F64, F32], ids=["f64", "f32"])
@pytest.mark.parametrize("kind,n", LENGTHS, ids=[lid(v) for v in LENGTHS])
def test_fft1d_per_line_accuracy(prec, kind, n):
    """each line on its own norm against long double: no line's error follows another line's magnitude"""
    N = n + 1 if kind == DST1 else n - 1
    s = acc_spec(prec, (1, 1, N), d=1)  # units of u sqrt(log2 N)
    a = max(8, min(64, (1 << 18) // n))
    x, sc = mixed((a, n), 0, prec, False, n)  # CONTIG: line i scaled by 1, 2^20, 2^-20, 0 in turn
    ref = sf.dct(x.astype(np.longdouble), type=1, axis=1) if kind == DCT1 else sf.dst(x.astype(np.longdouble), type=1, axis=1)
    got = on_device(lambda o, i: dfft.fft1d_r2r(prec, kind, dfft.FORWARD, n, a, 1, o, i), x, (a, n), RDT[prec])
    check_units("1D type-I CONTIG", s, got, ref, 0, sc, f"L={n}")
    b = 37
    x, sc = mixed((2, n, b), 2, prec, False, n + 1)  # TILED: column c scaled in turn
    ref = sf.dct(x.astype(np.longdouble), type=1, axis=1) if kind == DCT1 else sf.dst(x.astype(np.longdouble), type=1, axis=1)
    got = on_device(lambda o, i: dfft.fft1d_r2r(prec, kind, dfft.FORWARD, n, 2, b, o, i), x, (2, n, b), RDT[prec])
    check_units("1D type-I TILED", s, got, ref, 2, sc, f"L={n}")


# ---- one-rank plans -----------------------------------------------------------------------------------------------------
PLANS = [("slab", ("dct1",) * 3, (129, 129, 129), 3), ("zyx", ("dct1",) * 3, (129, 129, 129), 3), ("pencil", ("dct1",) * 3, (129, 129, 129), 3),
         ("slab", ("dct1",) * 3, (257, 257, 257), 3), ("slab", ("dct1", "r2hc", "r2hc"), (129, 128, 128), 3),
         ("zyx", ("dct1", "r2hc", "r2hc"), (129, 128, 128), 3), ("pencil", ("dct1", "r2hc", "r2hc"), (129, 128, 128), 3),
         ("slab", ("dst1",) * 3, (127, 255, 63), 3), ("pencil", ("dst1",) * 3, (127, 255, 63), 3), ("zyx", ("dst1",) * 3, (127, 255, 63), 3),
         ("slab", ("dst1", "dct", "dct1"), (63, 32, 65), 2), ("pencil", ("r2hc", "dst1", "dct1"), (16, 31, 33), 1)]


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("decomp,names,shape,d", PLANS)
def test_one_rank_plans(prec, decomp, names, shape, d):
    plan = make(names, prec, decomp, shape)
    kinds = kinds_of(names)
    assert plan.getR2RKinds() == kinds
    x = trand(shape, prec, 5)
    x0 = x.clone()
    osz = tuple(plan.getPartialSize(d))
    out = torch.full((int(np.prod(osz)) + 64,), 7.0, dtype=RDT[prec], device="cuda")
    plan.execR2R(out, x, dfft.FORWARD, d=d)
    got = out[:-64].reshape(osz)
    assert torch.equal(x, x0) and bool((out[-64:] == 7.0).all())
    xs = x.cpu().numpy().astype(np.float64)
    want = global_ref(xs, kinds, False, d)
    if d == 3 and len(set(kinds)) == 1:
        assert np.allclose(want, (sf.dctn if kinds[0] == DCT1 else sf.dstn)(xs, type=1))
    assert O.rel_l2(got.cpu().numpy(), want) < TOL[prec]
    back = torch.full((x.numel() + 64,), 7.0, dtype=RDT[prec], device="cuda")
    spec = got.clone()
    plan.execR2R(back, spec, dfft.INVERSE, d=d)
    assert torch.equal(spec, got) and bool((back[-64:] == 7.0).all())
    # the round trip scales by 2N per type-I axis (N = L - 1 for DCT-I, L + 1 for DST-I)
    assert O.rel_l2(back[:-64].reshape(shape).cpu().numpy() / round_trip_factor(names, shape, d), xs) < TOL[prec]
    plan.destroy()


def test_dct1_513_cube_on_device():
    """513^3 DCT-I in f64: a 16^3 sub-block of the spectrum from three contractions on the device, and the round trip"""
    names, shape = ("dct1",) * 3, (513, 513, 513)
    plan = make(names, F64, "slab", shape)
    x = trand(shape, F64, 8)
    y = torch.empty_like(x)
    plan.execR2R(y, x, dfft.FORWARD)
    ks = torch.arange(0, 513, 32, device="cuda", dtype=torch.float64)  # 17 modes per axis, k = 512 included
    j = torch.arange(513, device="cuda", dtype=torch.float64)
    Cm = torch.cos(math.pi * ks[:, None] * j[None, :] / 512) * 2
    Cm[:, 0] /= 2
    Cm[:, -1] /= 2  # DCT-I: x_0 + (-1)^k x_N + 2 sum_{n=1}^{N-1} x_n cos(pi n k / N)
    r = torch.tensordot(x, Cm, dims=([2], [1]))           # [513, 513, 17]
    r = torch.tensordot(r, Cm, dims=([1], [1]))           # [513, 17, 17]
    r = torch.tensordot(r, Cm, dims=([0], [1]))           # [17, 17, 17] over (z, y, x)
    r = r.permute(2, 1, 0)
    idx = ks.long()
    sub = y[idx][:, idx][:, :, idx]
    assert float(torch.linalg.norm(sub - r) / torch.linalg.norm(r)) < 1e-13
    back = torch.empty_like(x)
    plan.execR2R(back, y, dfft.INVERSE)
    back /= round_trip_factor(names, shape)
    assert float(torch.linalg.norm(back - x) / torch.linalg.norm(x)) < 1e-14
    plan.destroy()
    del x, y, back
    torch.cuda.empty_cache()


# ---- bit for bit --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("names", [("dct1", "r2hc", "r2hc"), ("dst1", "dst1", "dst1"), ("dct1", "dst", "dst1")])
def test_batch_inplace_scale_graph(prec, names):
    base = (16, 32, 64)
    shape = tuple(axis_len(n, KIND[k]) for n, k in zip(base, names))
    x = trand((3,) + shape, prec, 3)
    p3, p1 = make(names, prec, "slab", shape, batch=3), make(names, prec, "slab", shape)
    pin = make(names, prec, "slab", shape, batch=3, inplace=True)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        out = torch.empty_like(x)
        p3.execR2R(out, x, direction)
        for f in range(3):
            one = torch.empty_like(x[f])
            p1.execR2R(one, x[f].contiguous(), direction)
            assert torch.equal(out[f], one), ("batch", direction, f)
        field = pin.getDomainSize() // x.element_size()
        buf = torch.full((3 * field + 64,), 7.0, dtype=RDT[prec], device="cuda")
        for f in range(3):
            buf[f * field:f * field + x[f].numel()].copy_(x[f].reshape(-1))
        pin.execR2R(buf, buf, direction)
        for f in range(3):
            assert torch.equal(buf[f * field:f * field + x[f].numel()].reshape(shape), out[f]), ("in place", direction, f)
        assert bool((buf[-64:] == 7.0).all())
    # scale: the unscaled output times s, bit for bit
    n = round_trip_factor(names, shape)
    for direction in (dfft.FORWARD, dfft.INVERSE):
        plain = torch.empty_like(x[0])
        p1.setScale(1.0, 1.0)
        p1.execR2R(plain, x[0].contiguous(), direction)
        for s in (1.0 / n, 0.3):
            p1.setScale(s, s)
            scaled = torch.empty_like(plain)
            p1.execR2R(scaled, x[0].contiguous(), direction)
            assert torch.equal(scaled, plain * torch.tensor(s, dtype=RDT[prec], device="cuda")), (direction, s)
    p1.setScale(1.0, 1.0 / n)
    # graph replay of one-rank _async execs: the eager results, bit for bit
    xi = x[0].contiguous()
    y, back = torch.empty_like(xi), torch.empty_like(xi)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        p1.execR2R(y, xi, dfft.FORWARD, stream=st)
        p1.execR2R(back, y, dfft.INVERSE, stream=st)
    st.synchronize()
    assert O.rel_l2(back.cpu().numpy(), xi.cpu().numpy()) < TOL[prec]
    ey, eb = y.clone(), back.clone()
    y.zero_(); back.zero_()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cs = torch.cuda.current_stream()
        p1.execR2R(y, xi, dfft.FORWARD, stream=cs)
        p1.execR2R(back, y, dfft.INVERSE, stream=cs)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(y, ey) and torch.equal(back, eb)
    for p in (p3, p1, pin):
        p.destroy()


def test_timer_and_tune():
    shape = (33, 32, 31)
    p = make(("dct1", "r2hc", "dst1"), F64, "slab", shape)
    x = trand(shape, F64, 1)
    y = torch.empty_like(x)
    p.enableTimer(True)
    p.execR2R(y, x)
    steps = p.stepTimes()
    assert len(steps) == 3 and all(ms >= 0 for _, ms in steps)
    assert "sequential schedule" in p.tune(y, x)
    p.destroy()


# ---- multi-rank schedules with the real kernels --------------------------------------------------------------------------
REPLAYS = [  # P, decomp, base shape, p1, p2, comm, kinds
    (2, dfft.SLAB_ZY_THEN_X, (16, 16, 64), 2, 1, 0, (DCT1, DST1, DCT1)),
    (3, dfft.SLAB_ZY_THEN_X, (8, 16, 64), 3, 1, 1, (DCT1, R2HC, R2HC)),
    (4, dfft.SLAB_Z_THEN_YX, (16, 8, 32), 4, 1, 0, (DST1, DCT, DCT1)),
    (3, dfft.SLAB_Z_THEN_YX, (8, 4, 16), 3, 1, 1, (DCT1, DCT1, DST1)),
    (4, dfft.PENCIL, (8, 16, 32), 2, 2, 0, (DST1, DST1, DST1)),
    (6, dfft.PENCIL, (8, 16, 32), 2, 3, 1, (R2HC, DST1, DCT1)),
    (8, dfft.PENCIL, (16, 16, 1024), 4, 2, 0, (DCT1, DCT1, DCT1)),  # blocked second transposition with tails
    (5, dfft.SLAB_ZY_THEN_X, (16, 16, 128), 5, 1, 0, (DCT1, DST, DST1)),
]


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,base,p1,p2,comm,kinds", REPLAYS)
def test_multi_rank_replay(P, decomp, base, p1, p2, comm, kinds, inverse, prec):
    shape = tuple(axis_len(n, k) for n, k in zip(base, kinds))
    p = R.Plan(P, decomp, shape, p1, p2, kinds=kinds, prec=prec, comm=comm)
    x, _ = global_input(p, inverse, 3, 1)
    got = output(p, inverse, 3, x)
    want = global_ref(x[0].astype(np.float64), kinds, bool(inverse), 3)
    assert O.rel_l2(got[0].astype(np.float64), want) < TOL[prec]


# ---- physics ------------------------------------------------------------------------------------------------------------
def test_vertex_centred_dirichlet_poisson():
    """-Laplace u = f on the 63^3 interior nodes of a 64-cell grid with u = 0 on the boundary nodes: DST-I diagonalises the
    7-point Laplacian, eigenvalues -4 sin^2(pi k / 2N), k = 1..N-1; the residual of the solve is at round-off"""
    N = 64
    shape = (N - 1,) * 3
    plan = make(("dst1",) * 3, F64, "slab", shape)
    f = trand(shape, F64, 21)
    k = torch.arange(1, N, dtype=torch.float64, device="cuda")
    lk = -4 * torch.sin(math.pi * k / (2 * N)) ** 2
    lam = lk.view(-1, 1, 1) + lk.view(1, -1, 1) + lk.view(1, 1, -1)
    spec = torch.empty_like(f)
    plan.execR2R(spec, f, dfft.FORWARD)
    u = torch.empty_like(f)
    plan.execR2R(u, (spec / lam).contiguous(), dfft.INVERSE)
    u /= (2 * N) ** 3
    p = torch.nn.functional.pad(u, (1, 1, 1, 1, 1, 1))  # the boundary nodes: zero
    lap = (p[2:, 1:-1, 1:-1] + p[:-2, 1:-1, 1:-1] + p[1:-1, 2:, 1:-1] + p[1:-1, :-2, 1:-1] + p[1:-1, 1:-1, 2:] + p[1:-1, 1:-1, :-2] - 6 * u)
    err = float(torch.linalg.norm(lap - f) / torch.linalg.norm(f))
    assert err <= 1e-12, err
    plan.destroy()


@pytest.mark.parametrize("prec", [F64, F32])
def test_chebyshev_dct1(prec):
    """T_m(cos(pi j / N)) = cos(pi m j / N) on the Gauss-Lobatto points: its DCT-I is N delta_km, 2N at m = 0 and m = N"""
    N = 128
    j = torch.arange(N + 1, device="cuda", dtype=torch.float64)
    m = torch.arange(N + 1, device="cuda", dtype=torch.float64)
    T = torch.cos(m[:, None] * torch.arccos(torch.cos(math.pi * j[None, :] / N))).to(RDT[prec]).contiguous()  # [m][j]
    y = torch.empty_like(T)
    dfft.fft1d_r2r(prec, DCT1, dfft.FORWARD, N + 1, N + 1, 1, y, T)
    torch.cuda.synchronize()
    want = N * torch.eye(N + 1, dtype=torch.float64, device="cuda")
    want[0, 0] = want[N, N] = 2 * N
    err = float((y.double() - want).abs().max()) / (2 * N)
    assert err < (1e-13 if prec == F64 else 2e-5), err


def test_cpp_shim_type1_kinds(tmp_path):
    """tests/cpp/r2r1_shim_test.cpp: the shim constructor with type-I kinds and execR2R against the C ABI plan, by memcmp"""
    exe = str(tmp_path / "r2r1_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
                    os.path.join(HERE, "cpp", "r2r1_shim_test.cpp"), "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart",
                    "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
