"""Interleaved multi-component plans on one GPU: one-rank C2C plans against numpy on [X, Y, Z, C] tensors, bit-for-bit
comparisons with the batched plan on the permuted [C, X, Y, Z] input (512^3 x 3 included, where the batched plan runs the
fused z + y stage), scale, graph replay and batches, and 2-8 rank schedules replayed with the real kernels through
dfft_debug_run_step (gpu_replay.py)."""
import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from gpu_replay import output
from test_gpu_accuracy import check_units, ld, spec as unit_spec, unit_scales
from test_schedule_emulation import A2A, P2P, PE, SL, ZY

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

CLASSES = {SL: dfft.MPIcuFFT_Slab, ZY: dfft.MPIcuFFT_Slab_Z_Then_YX, PE: dfft.MPIcuFFT_Pencil}
TOL = {True: 1e-10, False: 1e-5}


def make(shape, comps, decomp=SL, f64=True, batch=1, transform="c2c"):
    plan = CLASSES[decomp](dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1) if decomp == PE else None, True, batch=batch, components=comps)
    return plan


def rand(shape, f64=True, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = torch.complex128 if f64 else torch.complex64
    return torch.randn(shape, dtype=dt, device="cuda", generator=g)


def exec_(plan, x, direction=dfft.FORWARD, d=3):
    out = torch.empty_like(x) if d == 3 else torch.empty(x.shape, dtype=x.dtype, device="cuda")
    plan.execC2C(out, x, direction, d)
    torch.cuda.synchronize()
    return out


def r2c(plan, x, d=3):
    """forward R2C of a real [X, Y, Z, C] tensor"""
    osz = plan.getPartialSize(d)
    out = torch.empty(tuple(osz) + (x.shape[-1],), dtype=torch.complex128 if x.dtype == torch.float64 else torch.complex64, device="cuda")
    plan.execR2C(out, x, d)
    torch.cuda.synchronize()
    return out


def c2r(plan, X):
    isz = plan.getInSize()
    out = torch.empty(tuple(isz) + (X.shape[-1],), dtype=torch.float64 if X.dtype == torch.complex128 else torch.float32, device="cuda")
    plan.execC2R(out, X)
    torch.cuda.synchronize()
    return out


def rel(a, b):
    return float(np.linalg.norm((a - b).ravel()) / np.linalg.norm(b.ravel()))


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("shape,comps,decomp", [((256, 256, 256), 3, SL), ((96, 128, 64), 5, SL), ((64, 32, 128), 17, ZY),
                                                ((32, 64, 16), 2, PE)])
def test_against_numpy(shape, comps, decomp, f64):
    plan = make(shape, comps, decomp, f64)
    assert plan.getComponents() == comps and plan.getInSize() == list(shape)
    x = rand(shape + (comps,), f64)
    y = exec_(plan, x)
    ref = np.fft.fftn(x.cpu().numpy().astype(np.complex128), axes=(0, 1, 2))
    assert rel(y.cpu().numpy(), ref) < TOL[f64]
    back = exec_(plan, y, dfft.INVERSE)
    n = shape[0] * shape[1] * shape[2]
    assert rel(back.cpu().numpy(), x.cpu().numpy() * n) < TOL[f64]
    plan.destroy()


@pytest.mark.parametrize("shape,comps,f64", [((64, 64, 64), 3, True), ((256, 256, 256), 3, True), ((512, 512, 512), 3, True),
                                             ((128, 64, 256), 5, False), ((32, 32, 64), 8, True), ((64, 32, 32), 17, True)])
def test_bit_identical_to_the_batched_plan(shape, comps, f64):
    """component c of the interleaved output equals, bit for bit, field c of the batched plan on the permuted input"""
    x = rand(shape + (comps,), f64, seed=1)
    ilv = make(shape, comps, f64=f64)
    bat = make(shape, 1, f64=f64, batch=comps)
    xp = x.permute(3, 0, 1, 2).contiguous()
    for direction in (dfft.FORWARD, dfft.INVERSE):
        a = exec_(ilv, x, direction)
        b = exec_(bat, xp, direction)
        assert torch.equal(a.permute(3, 0, 1, 2), b), direction
    ilv.destroy()
    bat.destroy()


@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("shape,comps,decomp", [((256, 256, 256), 3, SL), ((64, 64, 64), 2, SL), ((128, 64, 256), 7, SL),
                                                ((32, 64, 16), 5, ZY), ((64, 32, 32), 4, PE), ((16, 16, 8192), 3, SL)])
def test_r2c_against_numpy(shape, comps, decomp, f64):
    """the interleaved R2C / C2R z pass: forward against numpy's rfftn, inverse against irfftn, round trip, scale bit for bit"""
    plan = make(shape, comps, decomp, f64, transform="r2c")
    x = torch.randn(shape + (comps,), dtype=torch.float64 if f64 else torch.float32, device="cuda",
                    generator=torch.Generator(device="cuda").manual_seed(5))
    X = r2c(plan, x)
    ref = np.fft.rfftn(x.cpu().numpy().astype(np.float64), axes=(0, 1, 2))
    assert rel(X.cpu().numpy(), ref) < TOL[f64]
    n = shape[0] * shape[1] * shape[2]
    back = c2r(plan, X)
    assert rel(back.cpu().numpy(), x.cpu().numpy().astype(np.float64) * n) < TOL[f64]
    Xd = X.cpu().numpy().astype(np.complex128)
    assert rel(back.cpu().numpy(), np.fft.irfftn(Xd, s=shape, axes=(0, 1, 2)) * n) < TOL[f64]
    for d in (1, 2):
        refd = np.fft.rfft(x.cpu().numpy().astype(np.float64), axis=2)
        if d == 2:
            refd = np.fft.fft(refd, axis=1)
        assert rel(r2c(plan, x, d).cpu().numpy(), refd) < TOL[f64]
    plan.setScale(0.375, 1.5)
    assert torch.equal(r2c(plan, x), X * 0.375)
    assert torch.equal(c2r(plan, X), back * 1.5)
    plan.destroy()


def test_partial_scale_graph_and_batch():
    shape, comps = (64, 64, 128), 3
    plan = make(shape, comps)
    x = rand(shape + (comps,), seed=2)
    ref1 = np.fft.fft(x.cpu().numpy(), axis=2)
    assert rel(exec_(plan, x, d=1).cpu().numpy(), ref1) < 1e-10
    ref2 = np.fft.fftn(x.cpu().numpy(), axes=(1, 2))
    assert rel(exec_(plan, x, d=2).cpu().numpy(), ref2) < 1e-10
    y = exec_(plan, x)
    # scale: bit for bit the unscaled output times s
    plan.setScale(0.375, 1.0)
    ys = exec_(plan, x)
    assert torch.equal(ys, y * 0.375)
    plan.setScale(1.0, 1.0)
    # graph replay equals the eager exec
    out = torch.empty_like(x)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        plan.execC2C(out, x, dfft.FORWARD, stream=s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        plan.execC2C(out, x, dfft.FORWARD, stream=s)
    out.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, y)
    plan.destroy()
    # batch 2 x C 3 equals two separate execs
    pb = make(shape, comps, batch=2)
    xb = torch.stack([x, rand(shape + (comps,), seed=3)])
    yb = exec_(pb, xb)
    assert torch.equal(yb[0], y)
    one = make(shape, comps)
    assert torch.equal(yb[1], exec_(one, xb[1].contiguous()))
    pb.destroy()
    one.destroy()


# ---- multi-rank schedules on one GPU ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,comps", [
    (2, SL, (32, 32, 64), 2, 1, P2P, 3), (4, SL, (16, 24, 64), 4, 1, A2A, 5), (3, ZY, (12, 16, 32), 3, 1, P2P, 2), (3, ZY, (16, 16, 32), 3, 1, P2P, 2),
    (4, ZY, (16, 8, 32), 4, 1, A2A, 17), (4, PE, (16, 16, 64), 2, 2, P2P, 3), (8, PE, (16, 16, 32), 4, 2, A2A, 4),
    (6, PE, (12, 9, 64), 3, 2, P2P, 3)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_multi_rank_replay(P, decomp, shape, p1, p2, comm, comps, inverse):
    replay_case(P, decomp, shape, p1, p2, comm, comps, inverse, dfft.C2C)


@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,comps", [
    (2, SL, (32, 32, 64), 2, 1, P2P, 3), (4, SL, (16, 32, 64), 4, 1, A2A, 2), (3, SL, (16, 16, 64), 3, 1, P2P, 5),
    (3, ZY, (16, 16, 32), 3, 1, P2P, 7), (4, ZY, (16, 8, 32), 4, 1, A2A, 4), (4, PE, (16, 16, 64), 2, 2, P2P, 3),
    (8, PE, (16, 16, 32), 4, 2, A2A, 2), (6, PE, (16, 8, 64), 3, 2, P2P, 17)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_multi_rank_replay_r2c(P, decomp, shape, p1, p2, comm, comps, inverse):
    replay_case(P, decomp, shape, p1, p2, comm, comps, inverse, dfft.R2C)


def replay_case(P, decomp, shape, p1, p2, comm, comps, inverse, transform):
    """every rank's steps in lock step with the real kernels (gpu_replay.py, with the checks it makes of every plan);
    against numpy (R2C / C2R: each component against long double on its own norm) and, bit for bit, the one-rank plan"""
    d = 3
    c2c = transform == dfft.C2C
    one = make(shape, comps, decomp, transform="c2c" if c2c else "r2c")  # same decomposition: Z_Then_YX inverts y before x
    if c2c:
        x = rand(shape + (comps,), seed=4)
        spec = exec_(one, x)
        src, want = (spec, exec_(one, spec, dfft.INVERSE)) if inverse else (x, spec)
    else:
        # components of mixed magnitude (1, 2^20, 2^-20, 0, ...): each is held to the per-component long-double bound
        sc = unit_scales(comps)
        x = torch.randn(shape + (comps,), dtype=torch.float64, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
        x = x * torch.from_numpy(sc).cuda()
        spec = r2c(one, x)
        src, want = (spec, c2r(one, spec)) if inverse else (x, spec)
    p = R.Plan(P, decomp, shape, p1, p2, transform=transform, comm=comm, components=comps)
    full = output(p, inverse, d, src[None].cpu().numpy())[0]
    want = want.cpu().numpy()
    lay = lambda r, w: dfft.layout(decomp, transform, *shape, p1, p2, r, w)
    blk = lambda a, st, sz: a[st[0]:st[0] + sz[0], st[1]:st[1] + sz[1], st[2]:st[2] + sz[2]]
    for r in range(P):
        osz, ost = lay(r, 0 if inverse else d)
        got = blk(full, ost, osz)
        if not any(n & (n - 1) for n in shape):  # Bluestein passes: against the reference only
            assert np.array_equal(got, blk(want, ost, osz)), f"rank {r}"
        if c2c:
            ref = np.fft.ifftn(spec.cpu().numpy(), axes=(0, 1, 2)) * np.prod(shape) if inverse else np.fft.fftn(x.cpu().numpy(), axes=(0, 1, 2))
            assert rel(got, blk(ref, ost, osz)) < 1e-10
    if not c2c:
        ref = (np.fft.irfftn(ld(spec.cpu().numpy()), s=shape, axes=(0, 1, 2)) * np.prod(shape) if inverse
               else np.fft.rfftn(ld(x.cpu().numpy()), axes=(0, 1, 2)))
        check_units("replay R2C/C2R", unit_spec(dfft.F64, shape), full, ref, 3, sc, f"P={P} {'inv' if inverse else 'fwd'}")
    one.destroy()


def test_cpp_shim_interleaved(tmp_path):
    """tests/cpp/components_shim_test.cpp: MPIcuFFT_Slab<double>::initFFTInterleaved against the batched plan"""
    import os
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    exe = str(tmp_path / "components_shim_test")
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(root, "include"), "-I/usr/local/cuda/include", os.path.join(here, "cpp", "components_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
