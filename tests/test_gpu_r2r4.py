"""Type-IV real-to-real kinds (DCT-IV / DST-IV) on one GPU.

- dfft_fft1d_r2r with DFFT_DCT4 / DFFT_DST4 at every length, CONTIG and TILED, in place and out of place, against scipy's
  dct / dst(type=4); forward and inverse run the same transform.
- Per-line accuracy against long double at every length: lines of mixed magnitudes (1, 2^20, 2^-20, 0 in turn) held to the
  bounds of test_gpu_accuracy on each line's own norm, zero lines exact zeros.
- One-rank plans (slab, Z_Then_YX, pencil) against scipy's dctn / dstn(type=4) and the per-axis reference, partial d; round
  trips scale by 2N per type-IV axis; a 512^3 DCT-IV in f64 and f32.
- Bit for bit: in place against out of place, batch against single fields, scale against unscaled, graph replay against
  eager.
- 2-8 rank schedules replayed with the real kernels through dfft_debug_run_step (gpu_replay.py).
- A mixed-wall Poisson solve with (dct4, dst4, r2hc) on 32 x 64 x 128 cells (7-point Laplacian residual with the ghost
  rules of each wall).
- The C++ shim's per-axis constructor with type-IV kinds (tests/cpp/r2r4_shim_test.cpp)."""
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
from test_r2r4 import DCT, DST, R2HC, DCT1, DST1, DCT4, DST4, global_ref, r2r_1d, shape_for

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
KIND = {"dct": DCT, "dst": DST, "r2hc": R2HC, "dct1": DCT1, "dst1": DST1, "dct4": DCT4, "dst4": DST4}
F32, F64 = dfft.F32, dfft.F64
LENGTHS = [(k, 1 << l) for k in (DCT4, DST4) for l in range(2, 14)]


def lid(v):
    return f"{'dct4' if v[0] == DCT4 else 'dst4'}-{v[1]}"


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
        f *= {"r2hc": n, "dct": 2 * n, "dst": 2 * n, "dct1": 2 * (n - 1), "dst1": 2 * (n + 1), "dct4": 2 * n, "dst4": 2 * n}[k]
    return f


def type4_ref(x, kind, axis):
    return (sf.dct if kind == DCT4 else sf.dst)(x, type=4, axis=axis)


# ---- the single-axis call ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("kind,n", LENGTHS, ids=[lid(v) for v in LENGTHS])
def test_fft1d(prec, kind, n):
    for a, b in ((257 if n <= 256 else 7, 1), (3, 5), (2, 33), (1, 64)):  # CONTIG odd line count, TILED partial tiles
        x = np.random.default_rng(n + b).standard_normal((a, n, b)).astype(np.float64 if prec == F64 else np.float32)
        xin = torch.from_numpy(x).cuda()
        outs = []
        for direction in (dfft.FORWARD, dfft.INVERSE):
            out = torch.empty_like(xin)
            dfft.fft1d_r2r(prec, kind, direction, n, a, b, out, xin)
            torch.cuda.synchronize()
            assert O.rel_l2(out.cpu().numpy(), type4_ref(x.astype(np.float64), kind, 1)) < TOL[prec], (a, b, direction)
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
    s = acc_spec(prec, (1, 1, n), d=1)  # units of u sqrt(log2 N)
    a = max(8, min(64, (1 << 18) // n))
    x, sc = mixed((a, n), 0, prec, False, n)  # CONTIG: line i scaled by 1, 2^20, 2^-20, 0 in turn
    ref = type4_ref(x.astype(np.longdouble), kind, 1)
    got = on_device(lambda o, i: dfft.fft1d_r2r(prec, kind, dfft.FORWARD, n, a, 1, o, i), x, (a, n), RDT[prec])
    check_units("1D type-IV CONTIG", s, got, ref, 0, sc, f"N={n}")
    b = 37
    x, sc = mixed((2, n, b), 2, prec, False, n + 1)  # TILED: column c scaled in turn
    ref = type4_ref(x.astype(np.longdouble), kind, 1)
    got = on_device(lambda o, i: dfft.fft1d_r2r(prec, kind, dfft.FORWARD, n, 2, b, o, i), x, (2, n, b), RDT[prec])
    check_units("1D type-IV TILED", s, got, ref, 2, sc, f"N={n}")


# ---- one-rank plans -----------------------------------------------------------------------------------------------------
PLANS = [("slab", ("dct4",) * 3, (128, 128, 128), 3), ("zyx", ("dct4",) * 3, (128, 128, 128), 3), ("pencil", ("dct4",) * 3, (128, 128, 128), 3),
         ("slab", ("dct4", "r2hc", "r2hc"), (64, 128, 128), 3), ("zyx", ("dct4", "r2hc", "r2hc"), (64, 128, 128), 3),
         ("pencil", ("dct4", "r2hc", "r2hc"), (64, 128, 128), 3),
         ("slab", ("dst4",) * 3, (64, 256, 32), 3), ("pencil", ("dst4",) * 3, (64, 256, 32), 3), ("zyx", ("dst4",) * 3, (64, 256, 32), 3),
         ("slab", ("dst4", "dct", "dct1"), (64, 32, 65), 2), ("pencil", ("r2hc", "dst1", "dct4"), (16, 31, 32), 1),
         ("zyx", ("dct4", "dst4", "r2hc"), (32, 64, 128), 3), ("slab", ("dct1", "dct4", "dst4"), (17, 8, 4096), 3)]


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
        assert np.allclose(want, (sf.dctn if kinds[0] == DCT4 else sf.dstn)(xs, type=4))
    assert O.rel_l2(got.cpu().numpy(), want) < TOL[prec]
    back = torch.full((x.numel() + 64,), 7.0, dtype=RDT[prec], device="cuda")
    spec = got.clone()
    plan.execR2R(back, spec, dfft.INVERSE, d=d)
    assert torch.equal(spec, got) and bool((back[-64:] == 7.0).all())
    # the round trip scales by 2N per type-IV axis
    assert O.rel_l2(back[:-64].reshape(shape).cpu().numpy() / round_trip_factor(names, shape, d), xs) < TOL[prec]
    plan.destroy()


@pytest.mark.parametrize("prec", [F64, F32])
def test_dct4_512_cube(prec):
    """512^3 DCT-IV: against scipy's dctn(type=4), and the round trip"""
    names, shape = ("dct4",) * 3, (512, 512, 512)
    plan = make(names, prec, "slab", shape)
    x = trand(shape, prec, 8)
    y = torch.empty_like(x)
    plan.execR2R(y, x, dfft.FORWARD)
    want = sf.dctn(x.cpu().numpy().astype(np.float64), type=4, workers=-1)
    assert O.rel_l2(y.cpu().numpy(), want) < TOL[prec]
    del want
    back = torch.empty_like(x)
    plan.execR2R(back, y, dfft.INVERSE)
    back /= round_trip_factor(names, shape)
    assert float(torch.linalg.norm((back - x).double()) / torch.linalg.norm(x.double())) < TOL[prec]
    plan.destroy()
    del x, y, back
    torch.cuda.empty_cache()


# ---- bit for bit --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("names", [("dct4", "r2hc", "r2hc"), ("dst4", "dst4", "dst4"), ("dct4", "dst", "dst1")])
def test_batch_inplace_scale_graph(prec, names):
    shape = shape_for((16, 32, 64), kinds_of(names))
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
    shape = (32, 32, 33)
    p = make(("dct4", "r2hc", "dct1"), F64, "slab", shape)
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
    (2, dfft.SLAB_ZY_THEN_X, (16, 16, 64), 2, 1, 0, (DCT4, DST4, DCT4)),
    (3, dfft.SLAB_ZY_THEN_X, (8, 16, 64), 3, 1, 1, (DCT4, R2HC, R2HC)),
    (4, dfft.SLAB_Z_THEN_YX, (16, 8, 32), 4, 1, 0, (DST4, DCT, DCT1)),
    (3, dfft.SLAB_Z_THEN_YX, (8, 4, 16), 3, 1, 1, (DCT4, DCT4, DST4)),
    (4, dfft.PENCIL, (8, 16, 32), 2, 2, 0, (DST4, DST4, DST4)),
    (6, dfft.PENCIL, (8, 16, 32), 2, 3, 1, (R2HC, DST1, DCT4)),
    (8, dfft.PENCIL, (16, 16, 1024), 4, 2, 0, (DCT4, DCT4, DCT4)),  # blocked second transposition with tails
    (5, dfft.SLAB_ZY_THEN_X, (16, 16, 128), 5, 1, 0, (DCT4, DST, DST4)),
]


@pytest.mark.parametrize("prec", [F64, F32])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,base,p1,p2,comm,kinds", REPLAYS)
def test_multi_rank_replay(P, decomp, base, p1, p2, comm, kinds, inverse, prec):
    shape = shape_for(base, kinds)
    p = R.Plan(P, decomp, shape, p1, p2, kinds=kinds, prec=prec, comm=comm)
    x, _ = global_input(p, inverse, 3, 1)
    got = output(p, inverse, 3, x)
    want = global_ref(x[0].astype(np.float64), kinds, bool(inverse), 3)
    assert O.rel_l2(got[0].astype(np.float64), want) < TOL[prec]


# ---- physics ------------------------------------------------------------------------------------------------------------
def test_mixed_wall_poisson():
    """Laplace u = f on 32 x 64 x 128 cells: x Neumann at the low face and Dirichlet at the high one (DCT-IV), y Dirichlet /
    Neumann (DST-IV), z periodic (R2HC).  Each kind diagonalises the 3-point second difference with its ghost rules, so
    dividing by the sum of the per-axis eigenvalues solves the 7-point Laplacian; the residual is at round-off."""
    shape = (32, 64, 128)
    Nx, Ny, Nz = shape
    plan = make(("dct4", "dst4", "r2hc"), F64, "zyx", shape)
    f = trand(shape, F64, 21)

    def lam4(n):
        k = torch.arange(n, dtype=torch.float64, device="cuda")
        return -4 * torch.sin(math.pi * (2 * k + 1) / (4 * n)) ** 2

    kz = torch.arange(Nz, dtype=torch.float64, device="cuda")  # halfcomplex index k and N - k: the same eigenvalue
    lz = -4 * torch.sin(math.pi * kz / Nz) ** 2
    lam = lam4(Nx).view(-1, 1, 1) + lam4(Ny).view(1, -1, 1) + lz.view(1, 1, -1)
    spec = torch.empty_like(f)
    plan.execR2R(spec, f, dfft.FORWARD)
    u = torch.empty_like(f)
    plan.execR2R(u, (spec / lam).contiguous(), dfft.INVERSE)
    u /= 2 * Nx * 2 * Ny * Nz
    # ghost cells: x u_{-1} = u_0, u_N = -u_{N-1}; y u_{-1} = -u_0, u_N = u_{N-1}; z periodic
    px = torch.cat([u[:1], u, -u[-1:]], 0)
    py = torch.cat([-u[:, :1], u, u[:, -1:]], 1)
    pz = torch.cat([u[:, :, -1:], u, u[:, :, :1]], 2)
    lap = px[2:] + px[:-2] + py[:, 2:] + py[:, :-2] + pz[:, :, 2:] + pz[:, :, :-2] - 6 * u
    err = float(torch.linalg.norm(lap - f) / torch.linalg.norm(f))
    assert err <= 1e-10, err
    plan.destroy()


def test_cpp_shim_type4_kinds(tmp_path):
    """tests/cpp/r2r4_shim_test.cpp: the shim constructor with type-IV kinds and execR2R against the C ABI plan, by memcmp"""
    exe = str(tmp_path / "r2r4_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
                    os.path.join(HERE, "cpp", "r2r4_shim_test.cpp"), "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart",
                    "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
