"""Plans with strides (dfft_plan_set_strides) on the GPU.

One rank, every decomposition, through the Python execs on torch slices A[h:-h, h:-h, h:-h] of arrays with ghost layers:
C2C (power-of-two and Bluestein axes), R2C / C2R and R2R (DCT and a mixed (r2hc, dct1, dst4) plan), f64 and f32, at sizes
below the fused z + y stage, so that the plan without strides runs the same sequential schedule.  Each exec's interior must
equal that plan's output on dense tensors bit for bit: the passes are the same kernels over the same lines (the x pass's
y-z rows split into a1 x b keeps every line's arithmetic; TILED instantiations depend on the line length only at these
sizes).  The caller's whole input array and every output ghost element are unchanged, a scaled exec equals the unscaled one
times the scale bit for bit, and a CUDA graph of the _async execs replays what the eager execs computed.  A 512^3 C2C plan
with strides is checked against the fused plan without them within the oracle's tolerance.

Multi-rank plans run every rank's step list in lock step through dfft_debug_run_step with the real kernels (gpu_replay.py),
on caller arrays with poisoned ghost layers, bit for bit against the plan without strides replayed the same way."""
import os
import subprocess
from dataclasses import replace

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
import step_replay as R
import test_gpu_schedule_replay as G
from common import CDT, RDT, TOL
from gpu_replay import assemble, output, replay, same_bits

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C, DCT, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.R2HC
CLS = {SL: dfft.MPIcuFFT_Slab, ZY: dfft.MPIcuFFT_Slab_Z_Then_YX, PE: dfft.MPIcuFFT_Pencil}
PNAME = {dfft.F64: "double", dfft.F32: "float"}
HERE = os.path.dirname(os.path.abspath(__file__))
H = 2  # ghost layers


def halo_array(size, dtype, fill):
    """a [n0 + 2H][n1 + 2H][n2 + 2H] array of `fill` and its interior slice"""
    a = torch.full([n + 2 * H for n in size], fill, dtype=dtype, device="cuda")
    return a, a[H:-H, H:-H, H:-H]


def field_strides(t):
    return (t.shape[0] * t.stride(0),) + tuple(t.stride()[:2])


def new_plan(decomp, prec, transform, shape, in_strides=None, out_strides=None):
    f = CLS[decomp](dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=transform)
    part = dfft.Partition(1, 1) if decomp == PE else None
    f.initFFT(dfft.GlobalSize(*shape), part, True, in_strides=in_strides, out_strides=out_strides)
    return f


def execute(f, kind, out, in_, inverse, stream=None):
    if kind == "c2c":
        f.execC2C(out, in_, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)
    elif kind == "r2c":
        (f.execC2R if inverse else f.execR2C)(out, in_, stream=stream)
    else:
        f.execR2R(out, in_, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)


def same(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


CASES = [  # (id, transform name for the plan, exec kind, shape)
    ("c2c", "c2c", "c2c", (16, 32, 64)),
    ("bluestein", "c2c", "c2c", (12, 20, 24)),
    ("r2c", "r2c", "r2c", (16, 32, 64)),
    ("dct", "dct", "r2r", (16, 32, 64)),
    ("mixed", ("r2hc", "dct1", "dst4"), "r2r", (16, 33, 64)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("decomp", [SL, ZY, PE], ids=["slab", "zyx", "pencil"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_one_rank(case, decomp, prec):
    _, transform, kind, shape = case
    plain = new_plan(decomp, prec, transform, shape)
    phys_t = RDT[prec] if kind in ("r2c", "r2r") else CDT[prec]
    spec_t = RDT[prec] if kind == "r2r" else CDT[prec]
    nan = float("nan")
    a_phys, phys = halo_array(plain.getInSize(), phys_t, nan)   # the physical side's caller array
    a_spec, spec = halo_array(plain.getOutSize(), spec_t, nan)  # the spectral side's
    f = new_plan(decomp, prec, transform, shape, field_strides(phys), field_strides(spec))
    assert f.getStrides() == (field_strides(phys), field_strides(spec))
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(plain.getInSize(), dtype=phys_t, device="cuda", generator=g)
    phys.copy_(x)
    # forward: the interior of the output array against the plan without strides, nothing else touched
    want = torch.empty(plain.getOutSize(), dtype=spec_t, device="cuda")
    execute(plain, kind, want, x, False)
    before = a_phys.clone()
    execute(f, kind, spec, phys, False)
    torch.cuda.synchronize()
    assert same(spec, want)
    assert same(a_phys, before), "the input array changed"
    ghost = torch.ones_like(a_spec, dtype=torch.bool)
    ghost[H:-H, H:-H, H:-H] = False
    assert torch.isnan(a_spec[ghost]).all(), "an output ghost element was written"
    # inverse from the spectrum, into the physical array's interior
    back = torch.empty_like(x)
    execute(plain, kind, back, want, True)
    before = a_spec.clone()
    phys.fill_(0)
    execute(f, kind, phys, spec, True)
    torch.cuda.synchronize()
    assert same(phys, back)
    assert same(a_spec, before)
    ghost = torch.ones_like(a_phys, dtype=torch.bool)
    ghost[H:-H, H:-H, H:-H] = False
    assert torch.isnan(a_phys[ghost]).all(), "an input-side ghost element was written by the inverse"
    # scale: the unscaled output times s, bit for bit
    s = 0.37
    f.setScale(s, s)
    execute(f, kind, spec, phys.copy_(x), False)
    r = want.real.dtype if want.is_complex() else want.dtype
    sv = torch.tensor(s, dtype=r, device="cuda")
    scaled = torch.view_as_complex(torch.view_as_real(want) * sv) if want.is_complex() else want * sv
    assert same(spec, scaled)
    f.setScale(1.0, 1.0)
    # torch slices with other strides, or dense tensors, are refused
    with pytest.raises(ValueError):
        execute(f, kind, spec, x, False)
    with pytest.raises(ValueError):
        wider = torch.zeros([n + 2 * H + 2 for n in plain.getInSize()], dtype=phys_t, device="cuda")
        execute(f, kind, spec, wider[H + 1:-H - 1, H + 1:-H - 1, H + 1:-H - 1], False)  # the block's shape, other strides
    with pytest.raises(ValueError):
        execute(f, kind, spec, a_phys[H:-H, H:-H, :], False)
    # graph replay of the _async execs against eager ones
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        execute(f, kind, spec, phys.copy_(x), False, stream=st)
        execute(f, kind, phys, spec, True, stream=st)
    st.synchronize()
    eager_spec, eager_phys = spec.clone(), phys.clone()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        cs = torch.cuda.current_stream()
        execute(f, kind, spec, phys, False, stream=cs)
        execute(f, kind, phys, spec, True, stream=cs)
    phys.copy_(x)
    spec.zero_()
    gr.replay()
    torch.cuda.synchronize()
    assert same(spec, eager_spec) and same(phys, eager_phys)
    f.destroy()
    plain.destroy()


@pytest.mark.gpu
def test_batched_and_partial_one_rank():
    """batch 2 with fields further apart than the arrays, and the partial execs (physical side with strides, the spectral
    side of d < 3 dense)"""
    shape, prec = (16, 32, 64), dfft.F64
    plain = CLS[SL](dfft.Configurations(), dfft.Comm(), precision="double", transform="c2c")
    plain.initFFT(dfft.GlobalSize(*shape), None, True, batch=2)
    big = torch.full((2 * (16 + 2 * H + 1), 32 + 2 * H, 64 + 2 * H), float("nan"), dtype=CDT[prec], device="cuda")
    ps, rs = big.stride(0), big.stride(1)
    a = big.as_strided((2,) + shape, ((16 + 2 * H + 1) * ps, ps, rs, 1), H * ps + H * rs + H)  # fields 16 + 2H + 1 planes apart
    st = (a.stride(0), a.stride(1), a.stride(2))
    f = CLS[SL](dfft.Configurations(), dfft.Comm(), precision="double", transform="c2c")
    f.initFFT(dfft.GlobalSize(*shape), None, True, batch=2, in_strides=st)
    x = torch.randn((2,) + shape, dtype=CDT[prec], device="cuda")
    a.copy_(x)
    before = big.clone()
    for d in (1, 2, 3):
        want = torch.empty((2,) + tuple(plain.getPartialSize(d)), dtype=CDT[prec], device="cuda")
        plain.execC2C(want, x, dfft.FORWARD, d=d)
        got = torch.empty_like(want)
        f.execC2C(got, a, dfft.FORWARD, d=d)
        assert same(got, want) and same(big, before), d
        back = torch.empty_like(x)
        plain.execC2C(back, want, dfft.INVERSE, d=d)
        a.zero_()
        f.execC2C(a, want, dfft.INVERSE, d=d)
        assert same(a, back), d
        a.copy_(x)
    f.destroy()
    plain.destroy()


@pytest.mark.gpu
def test_tune_has_one_candidate():
    shape = (16, 32, 64)
    a, phys = halo_array(shape, torch.complex128, 0.0)
    f = new_plan(SL, dfft.F64, "c2c", shape, field_strides(phys), None)
    out = torch.empty(shape, dtype=torch.complex128, device="cuda")
    assert "plans with strides run the sequential schedule" in f.tune(out, phys)
    f.destroy()


@pytest.mark.gpu
def test_512_cubed_against_the_fused_plan():
    """the embedded plan runs the sequential schedule; the plan without strides the fused z + y stage"""
    shape = (512, 512, 512)
    plain = new_plan(SL, dfft.F64, "c2c", shape)
    x = torch.randn(shape, dtype=torch.complex128, device="cuda")
    want = torch.empty_like(x)
    plain.execC2C(want, x, dfft.FORWARD)
    del plain
    torch.cuda.empty_cache()
    a_in, phys = halo_array(shape, torch.complex128, 0.0)
    phys.copy_(x)
    del x
    a_out, spec = halo_array(shape, torch.complex128, float("nan"))
    f = new_plan(SL, dfft.F64, "c2c", shape, field_strides(phys), field_strides(spec))
    f.execC2C(spec, phys, dfft.FORWARD)
    torch.cuda.synchronize()
    rel = float(torch.linalg.vector_norm(spec - want) / torch.linalg.vector_norm(want))
    assert rel < TOL[dfft.F64], rel
    assert torch.isnan(a_out[:H]).all() and torch.isnan(a_out[-H:]).all()
    f.destroy()


# ---- multi-rank plans with the real kernels ---------------------------------------------------------------------------------
def check_multi(p, inverse, d=3, seed=0):
    """p's replay (H ghost layers around each block of its embedded sides) against the plan without strides, bit for bit"""
    x, _ = G.global_input(p, inverse, d, seed)
    got = output(p, inverse, d, x)
    want = assemble(replay(replace(p, embed=None), inverse, d, x))
    assert same_bits(got, want), f"differs from the plan without strides at {np.argwhere(got != want)[:8].tolist()}"
    return x, got


def multi(P, decomp, transform, shape, p1, p2, comm=0, embed="both", **kw):
    return R.Plan(P, decomp, shape, p1, p2, transform=transform, comm=comm, embed=embed, halo=H, **kw)


MULTI = [
    # (id, P, decomp, transform, shape, p1, p2, kinds)
    ("slab3", 3, SL, C2C, (8, 8, 16), 3, 1, None),
    ("zyx3", 3, ZY, C2C, (8, 8, 16), 3, 1, None),
    ("pencil2x2", 4, PE, C2C, (8, 8, 16), 2, 2, None),
    ("pencil2x3", 6, PE, C2C, (8, 8, 16), 2, 3, None),
    ("pencil2x4", 8, PE, C2C, (8, 8, 8), 2, 4, None),
    ("slab2-bluestein", 2, SL, C2C, (6, 12, 10), 2, 1, None),
    ("pencil-r2c", 4, PE, R2C, (8, 8, 16), 2, 2, None),
    ("zyx3-r2c", 3, ZY, R2C, (8, 8, 16), 3, 1, None),
    ("slab3-dct", 3, SL, None, (8, 8, 16), 3, 1, (DCT, DCT, DCT)),
    ("pencil-mixed", 4, PE, None, (8, 9, 8), 2, 2, (R2HC, dfft.DCT1, dfft.DST4)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("comm", [0, 1], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("case", MULTI, ids=[c[0] for c in MULTI])
def test_multi_rank(case, inv, comm):
    _, P, decomp, transform, shape, p1, p2, kinds = case
    check_multi(multi(P, decomp, transform, shape, p1, p2, comm, kinds=kinds), inv)


@pytest.mark.gpu
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("decomp,P,p1,p2,nz", [(SL, 3, 3, 1, 18), (PE, 4, 2, 2, 36)], ids=["slab", "pencil"])
def test_multi_rank_blocked_tails(decomp, P, p1, p2, nz, inv, monkeypatch):
    monkeypatch.setenv("DFFT_BLOCKED", "4")
    check_multi(multi(P, decomp, C2C, (8, 8, nz), p1, p2), inv)


@pytest.mark.gpu
@pytest.mark.parametrize("embed", ["in", "out", "both"])
def test_multi_rank_batch_gap_scale(embed):
    for inv in (0, 1):
        x, plain = check_multi(multi(4, PE, C2C, (8, 8, 16), 2, 2, embed=embed, batch=2, gap=6), inv)
        _, scaled = check_multi(multi(4, PE, C2C, (8, 8, 16), 2, 2, embed=embed, batch=2, gap=6, scale=(0.37, 1 / 96)), inv)
        r = plain.real.dtype
        want = (np.ascontiguousarray(plain).view(r) * r.type((0.37, 1 / 96)[inv])).view(plain.dtype)
        assert same_bits(scaled, want)


@pytest.mark.gpu
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("decomp,p1,p2", [(SL, 4, 1), (PE, 2, 2)], ids=["slab", "pencil"])
def test_multi_rank_partial(decomp, p1, p2, d, inv):
    check_multi(multi(4, decomp, C2C, (8, 8, 16), p1, p2), inv, d)


@pytest.mark.gpu
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
def test_multi_rank_x_kept(inv):
    check_multi(multi(4, PE, C2C, (8, 8, 16), 2, 2, axes=(0, 1, 1)), inv)


@pytest.mark.gpu
def test_cpp_shim(tmp_path):
    """tests/cpp/embedded_shim_test.cpp: the shim's setStrides and one rank's execs on arrays with ghost layers"""
    exe = str(tmp_path / "embedded_shim_test")
    root = os.path.dirname(HERE)
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), "-I/usr/local/cuda/include",
                    os.path.join(HERE, "cpp", "embedded_shim_test.cpp"), "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64",
                    "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
