"""16-bit plans (DFFT_F16 / DFFT_BF16) on one H100.

The 16-bit passes run the f32 kernels' arithmetic on values widened from 16 bits and round once as they store, so they
have an exact reference: the f32 pass on the widened input, times the pass's factor in f32, rounded to 16 bits by torch
(round to nearest even, like __float22half2_rn / __float22bfloat162_rn).
  - kernels: dfft_fft1d_contig (C2C, R2C, C2R) and dfft_fft1d_strided at every length against that reference, bit for bit;
  - one-rank plans: the exec against the composition of f32 single-axis passes in the schedule's axis order, bit for bit;
  - accuracy: 256^3 and 512^3 against the float64 transform of the widened input, and round trips;
  - the scale split: an FP16 512^3 forward of a constant field is exact with (1/N, 1) and overflows unscaled, as documented;
  - multi-rank schedules: the one-GPU lock-step replay (gpu_replay.py) of 2..8 ranks equals the one-rank replay bit for bit;
  - graph capture, the timer, dfft_plan_tune, the Python binding with torch.complex32 and the C++ shim."""
from __future__ import annotations

import math
import os
import subprocess

import numpy as np
import pytest

import distributedfft_b200 as dfft
import gpu_replay as G
import step_replay as R

torch = pytest.importorskip("torch")

F16, BF16, F32 = dfft.F16, dfft.BF16, dfft.F32
HT = {F16: torch.float16, BF16: torch.bfloat16}
NAME = {F16: "half", BF16: "bfloat16"}
TOL = {F16: 2e-3, BF16: 1.6e-2}
FWD, INV = dfft.FORWARD, dfft.INVERSE


def bits(t):
    return t.contiguous().view(torch.int16)


def assert_same(got, want, what):
    g, w = bits(got).reshape(-1), bits(want).reshape(-1)
    if not torch.equal(g, w):
        bad = (g != w).nonzero().flatten()
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.numel()} of {g.numel()} 16-bit values differ; first at {i}: bits {int(g[i])} != {int(w[i])}")


def rnd(shape, prec, gen, sigma=1.0):
    return (torch.randn(*shape, generator=gen, device="cuda") * sigma).to(HT[prec])


# ---- kernels -------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("l", range(1, 14))
def test_kernels_equal_rounded_f32_kernels(prec, l):
    g = torch.Generator(device="cuda").manual_seed(100 + l)
    n = 1 << l
    H = HT[prec]
    lines = max(3, (1 << 17) >> l) + 1  # one CTA's lines not full
    for direction in (FWD, INV):
        x = rnd((lines, n, 2), prec, g)
        got, ref = torch.full_like(x, float("nan")), torch.empty(lines, n, 2, device="cuda")
        dfft.fft1d_contig(prec, 0, direction, n, lines, got, n, x, n)
        dfft.fft1d_contig(F32, 0, direction, n, lines, ref, n, x.float(), n)
        torch.cuda.synchronize()
        assert_same(got, ref.to(H), f"contig n={n} dir={direction}")
        a, b = 3, 37  # rows that fill no whole tile
        x = rnd((a, n, b, 2), prec, g)
        got, ref = torch.full_like(x, float("nan")), torch.empty(a, n, b, 2, device="cuda")
        dfft.fft1d_strided(prec, direction, a, n, b, got, x)
        dfft.fft1d_strided(F32, direction, a, n, b, ref, x.float())
        torch.cuda.synchronize()
        assert_same(got, ref.to(H), f"strided n={n} dir={direction}")
    # R2C / C2R: lines of 2n reals through n-point complex lines
    nr = 2 * n
    xr = rnd((lines, nr), prec, g)
    spec, ref = torch.full((lines, n + 1, 2), float("nan"), dtype=H, device="cuda"), torch.empty(lines, n + 1, 2, device="cuda")
    dfft.fft1d_contig(prec, 1, FWD, nr, lines, spec, n + 1, xr, nr)
    dfft.fft1d_contig(F32, 1, FWD, nr, lines, ref, n + 1, xr.float(), nr)
    torch.cuda.synchronize()
    assert_same(spec, ref.to(H), f"r2c n={nr}")
    back, refb = torch.full((lines, nr), float("nan"), dtype=H, device="cuda"), torch.empty(lines, nr, device="cuda")
    dfft.fft1d_contig(prec, 2, INV, nr, lines, back, nr, spec.clone(), n + 1)
    dfft.fft1d_contig(F32, 2, INV, nr, lines, refb, nr, spec.float(), n + 1)
    torch.cuda.synchronize()
    assert_same(back, refb.to(H), f"c2r n={nr}")


# ---- one-rank plans, bit for bit -------------------------------------------------------------------------------------------
def make_plan(prec, transform, shape, scale=(1.0, 1.0), cls=None, partition=None, **init):
    plan = (cls or dfft.MPIcuFFT_Slab)(dfft.Configurations(), dfft.Comm(0, 1, None, 0), precision=NAME[prec], transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), partition, True, **init)
    plan.setScale(*scale)
    return plan


def factors(plan, inverse, d=3):
    """{axis letter: factor} of the plan's FFT passes (1 where the describe lists none)"""
    sc = __import__("json").loads(R.describe_raw(plan._h, inverse, d))
    f = {}
    for st in sc["steps"]:
        if st["type"] == 0 and st["kind"] not in (6, 7):
            f[st["label"][0]] = st.get("factor", 1.0)
    return f


def f32_pass(prec, axis, kind, direction, x16, dims, factor):
    """one f32 single-axis pass over the widened 16-bit array x16 ([nx, ny, nzc, 2]; real [nx, ny, nz] for R2C's input),
    times factor in f32, rounded to 16 bits"""
    nx, ny, nz = dims
    xf = x16.float()
    if axis == 2 and kind == 1:  # R2C: nz reals -> nz/2 + 1 points
        out = torch.empty(nx, ny, nz // 2 + 1, 2, device="cuda")
        dfft.fft1d_contig(F32, 1, FWD, nz, nx * ny, out, nz // 2 + 1, xf, nz)
    elif axis == 2 and kind == 2:
        out = torch.empty(nx, ny, nz, device="cuda")
        dfft.fft1d_contig(F32, 2, INV, nz, nx * ny, out, nz, xf, nz // 2 + 1)
    else:
        out = torch.empty_like(xf)
        nzc = xf.shape[2]
        if axis == 2:
            dfft.fft1d_contig(F32, 0, direction, nz, nx * ny, out, nz, xf, nz)
        elif axis == 1:
            dfft.fft1d_strided(F32, direction, nx, ny, nzc, out, xf)
        else:
            dfft.fft1d_strided(F32, direction, 1, nx, ny * nzc, out, xf)
    torch.cuda.synchronize()
    if factor != 1.0:
        out = out * torch.tensor(factor, dtype=torch.float32, device="cuda")
    return out.to(HT[prec])


def composed(prec, transform, shape, inverse, x16, f):
    c2c = transform == "c2c"
    order = "xyz" if inverse else "zyx"
    y = x16
    for a in order:
        axis = "xyz".index(a)
        kind = 0 if c2c or axis != 2 else (2 if inverse else 1)
        y = f32_pass(prec, axis, kind, INV if inverse else FWD, y, shape, f[a])
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("shape", [(64, 64, 64), (256, 128, 64)], ids=["64c", "256x128x64"])
def test_plan_equals_composed_f32_passes(prec, transform, shape):
    g = torch.Generator(device="cuda").manual_seed(7)
    nx, ny, nz = shape
    N = nx * ny * nz
    c2c = transform == "c2c"
    nzc = nz if c2c else nz // 2 + 1
    for scale in ((1.0, 1.0), (1.0 / N, 1.0), (-3.0, 0.5)):
        plan = make_plan(prec, transform, shape, scale)
        for inverse in (0, 1):
            f = factors(plan, inverse)
            assert set(f) == set("xyz")
            if scale[inverse] == 1.0:
                assert all(v == 1.0 for v in f.values())
            if scale[inverse] == 1.0 / N:
                assert f == {"x": 1.0 / nx, "y": 1.0 / ny, "z": 1.0 / nz}
            last = "z" if inverse else "x"
            assert all((v < 0) == (a == last and scale[inverse] < 0) for a, v in f.items())
            if inverse:
                x = rnd((nx, ny, nzc, 2), prec, g)
                out = torch.full((nx, ny, nz, 2) if c2c else (nx, ny, nz), float("nan"), dtype=HT[prec], device="cuda")
                plan.execC2C(out, x, INV) if c2c else plan.execC2R(out, x.clone())
            else:
                x = rnd((nx, ny, nz, 2) if c2c else (nx, ny, nz), prec, g)
                out = torch.full((nx, ny, nzc, 2), float("nan"), dtype=HT[prec], device="cuda")
                plan.execC2C(out, x, FWD) if c2c else plan.execR2C(out, x)
            torch.cuda.synchronize()
            assert_same(out, composed(prec, transform, shape, inverse, x, f), f"{transform} {shape} scale={scale} inverse={inverse}")
        plan.destroy()


# ---- accuracy against float64 ----------------------------------------------------------------------------------------------
def cplx(t):
    return torch.view_as_complex(t.double()) if t.shape[-1] == 2 and t.dim() == 4 else t.double()


def rel(a, b):
    return float(torch.linalg.vector_norm(a - b) / torch.linalg.vector_norm(b))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("n", [256, 512])
def test_accuracy_against_float64(prec, transform, n):
    g = torch.Generator(device="cuda").manual_seed(11)
    shape = (n, n, n)
    N = n ** 3
    c2c = transform == "c2c"
    plan = make_plan(prec, transform, shape, (1.0, 1.0 / N))
    # sigma 1/4: the largest unnormalised 512^3 output stays well inside FP16's range
    x = rnd(shape + ((2,) if c2c else ()), prec, g, 0.25)
    spec = torch.empty(n, n, n if c2c else n // 2 + 1, 2, dtype=HT[prec], device="cuda")
    plan.execC2C(spec, x, FWD) if c2c else plan.execR2C(spec, x)
    back = torch.empty_like(x)
    plan.execC2C(back, spec, INV) if c2c else plan.execC2R(back, spec.clone())
    torch.cuda.synchronize()
    xd = cplx(x)
    ref = torch.fft.fftn(xd) if c2c else torch.fft.rfftn(xd)
    e_fwd = rel(cplx(spec), ref)
    del ref
    e_rt = rel(cplx(back), xd)
    print(f"{NAME[prec]} {transform} {n}^3: forward rel-L2 {e_fwd:.3e}, round trip {e_rt:.3e}")
    assert e_fwd <= TOL[prec] and e_rt <= TOL[prec], (e_fwd, e_rt)
    plan.destroy()


# ---- the scale split and FP16's range --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_fp16_constant_field_scale_split():
    n = 512
    one = torch.zeros(n, n, n, 2, dtype=torch.float16, device="cuda")
    one[..., 0] = 1.0
    out = torch.empty_like(one)
    plan = make_plan(F16, "c2c", (n, n, n), (1.0 / n ** 3, 1.0))
    plan.execC2C(out, one, FWD)
    torch.cuda.synchronize()
    o = out.float()
    assert torch.isfinite(o).all()
    assert o[0, 0, 0, 0].item() == 1.0 and o[0, 0, 0, 1].item() == 0.0
    o[0, 0, 0, 0] = 0.0
    assert not o.any(), "every bin but DC is exactly 0"
    # unscaled: the y pass stores 512^2 = 262144 at the (y, z) DC of every x plane, beyond FP16's 65504
    plan.setScale(1.0, 1.0)
    plan.execC2C(out, one, FWD, d=2)
    torch.cuda.synchronize()
    o = out.float()
    assert (o[:, 0, 0, 0] == float("inf")).all() and not o[:, 0, 0, 1].any()
    o[:, 0, 0, 0] = 0.0
    assert not o.any()
    plan.execC2C(out, one, FWD)
    torch.cuda.synchronize()
    assert not math.isfinite(out[0, 0, 0, 0].float().item())
    plan.destroy()


# ---- multi-rank schedules on one GPU ---------------------------------------------------------------------------------------
SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
REPLAYS = [
    # P, decomp, shape, p1, p2, comm, batch, inplace, axes, d
    (2, SL, (16, 32, 64), 2, 1, 0, None, False, None, 3),
    (4, SL, (16, 32, 64), 4, 1, 1, None, False, None, 3),
    (4, ZY, (16, 32, 64), 4, 1, 0, None, False, None, 3),
    (4, ZY, (16, 32, 64), 4, 1, 1, None, False, None, 3),
    (4, PE, (16, 32, 64), 2, 2, 0, None, False, None, 3),
    (8, PE, (16, 32, 64), 2, 4, 1, None, False, None, 3),
    (8, PE, (16, 32, 64), 2, 4, 0, None, False, None, 2),      # partial d
    (4, SL, (16, 32, 64), 4, 1, 0, 2, False, None, 3),         # batch 2
    (4, PE, (16, 32, 64), 2, 2, 0, None, True, None, 3),       # in place
    (4, SL, (16, 32, 64), 4, 1, 1, None, True, None, 3),
    (4, PE, (16, 32, 64), 2, 2, 0, None, False, (0, 1, 1), 3),  # kept x axis
]


def packed(x16):
    """[..., 2] 16-bit pairs -> the uint32 elements gpu_replay moves"""
    return np.ascontiguousarray(x16.cpu().view(torch.int16).numpy()).view(np.uint32)[..., 0]


def unpacked(u, prec):
    return torch.from_numpy(np.ascontiguousarray(u).view(np.int16).reshape(u.shape + (2,))).view(HT[prec])


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", REPLAYS, ids=lambda c: f"P{c[0]}-{'sl zy pe'.split()[c[1]]}-{'a2a' if c[5] else 'p2p'}-d{c[9]}"
                         + ("-b2" if c[6] else "") + ("-ip" if c[7] else "") + ("-keepx" if c[8] else ""))
def test_replay_of_ranks_equals_one_rank(prec, case):
    P, decomp, shape, p1, p2, comm, batch, inplace, axes, d = case
    g = torch.Generator(device="cuda").manual_seed(3)
    fields = batch or 1
    x = [packed(rnd(shape + (2,), prec, g)) for _ in range(fields)]
    for inverse in (0, 1):
        scale = (1.0, -1.0 / 4096) if inverse else (1.0 / 2048, 1.0)
        plan = lambda P_, decomp_, p1_, p2_: R.Plan(P_, decomp_, shape, p1_, p2_, transform=dfft.C2C, prec=prec, comm=comm, batch=batch,
                                                    inplace=inplace, axes=axes, scale=scale)
        got = G.assemble(G.replay(plan(P, decomp, p1, p2), inverse, d, x))
        again = G.assemble(G.replay(plan(P, decomp, p1, p2), inverse, d, x, descending=True))
        one = G.assemble(G.replay(plan(1, decomp, 1, 1), inverse, d, x))
        assert not torch.isnan(unpacked(got, prec).float()).any(), "output elements never written"
        assert G.same_bits(again, got), "the result depends on the order of the ranks within a step"
        assert G.same_bits(got, one), f"inverse={inverse}: {int((got != one).sum())} elements differ from the one-rank plan"


# ---- options -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
def test_graph_capture_timer_and_tune(prec):
    shape = (64, 64, 64)
    g = torch.Generator(device="cuda").manual_seed(9)
    plan = make_plan(prec, "c2c", shape, (1.0 / 64 ** 3, 1.0))
    x = rnd(shape + (2,), prec, g)
    out = torch.empty_like(x)
    s = torch.cuda.current_stream()
    plan.execC2C(out, x, FWD, stream=s)  # eager: sets the kernels up
    torch.cuda.synchronize()
    eager = out.clone()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        plan.execC2C(out, x, FWD, stream=torch.cuda.current_stream())
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    assert_same(out, eager, "graph replay")
    plan.enableTimer(True)
    plan.execC2C(out, x, FWD)
    torch.cuda.synchronize()
    labels = [l for l, _ in plan.stepTimes()]
    assert plan.lastLaunchCount() >= 3 and labels and all(t >= 0 for _, t in plan.stepTimes())
    assert_same(out, eager, "timed exec")
    report = plan.tune(out, x, FWD)
    assert "16-bit" in report and "overlapped" not in report, report
    plan.destroy()


@pytest.mark.gpu
def test_python_binding_complex32_end_to_end():
    shape = (32, 64, 128)
    N = math.prod(shape)
    x = (torch.randn(shape, dtype=torch.complex64, device="cuda")).to(torch.complex32)
    plan = make_plan(F16, "c2c", shape, (1.0 / N, 1.0))
    out = torch.empty_like(x)
    plan.execC2C(out, x, FWD)
    back = torch.empty_like(x)
    plan.execC2C(back, out, INV)
    torch.cuda.synchronize()
    ref = torch.fft.fftn(x.to(torch.complex128)) / N
    assert rel(out.to(torch.complex128), ref) < TOL[F16]
    assert rel(back.to(torch.complex128), x.to(torch.complex128)) < TOL[F16]
    plan.destroy()
    # R2C: torch.float16 on the real side, torch.complex32 on the complex one
    xr = torch.randn(shape, device="cuda").half()
    plan = make_plan(F16, "r2c", shape)
    spec = torch.empty(shape[0], shape[1], shape[2] // 2 + 1, dtype=torch.complex32, device="cuda")
    plan.execR2C(spec, xr)
    torch.cuda.synchronize()
    assert rel(spec.to(torch.complex128), torch.fft.rfftn(xr.double())) < TOL[F16]
    plan.destroy()
    # BF16: a trailing dimension of 2 on the complex side
    xb = torch.randn(shape + (2,), device="cuda").bfloat16()
    plan = make_plan(BF16, "c2c", shape, (1.0 / N, 1.0))
    outb = torch.empty_like(xb)
    plan.execC2C(outb, xb, FWD)
    torch.cuda.synchronize()
    assert rel(torch.view_as_complex(outb.double()), torch.fft.fftn(torch.view_as_complex(xb.double())) / N) < TOL[BF16]
    plan.destroy()


@pytest.mark.gpu
def test_cpp_shim_half(tmp_path):
    """tests/cpp/half_shim_test.cpp: MPIcuFFT_Slab<__half> and MPIcuFFT_Pencil<__nv_bfloat16> against the C ABI plans, memcmp"""
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    exe = str(tmp_path / "half_shim_test")
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), "-I/usr/local/cuda/include", os.path.join(here, "cpp", "half_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
