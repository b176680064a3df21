"""In-place plans on one GPU: the output of an in-place exec equals the out-of-place plan's output bit for bit (same kernels,
same arithmetic), nothing beyond the buffer is touched, out != in is refused, graph replays match eager execs, and a
2048 x 1024 x 1024 complex-double grid — 128 GiB out of place — transforms in place on one 80 GB H100."""
import ctypes as C
import os
import subprocess

import pytest

import distributedfft_b200 as dfft
from distributedfft_b200._lib import DfftError, lib

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CANARY = 4096  # bytes after the buffer that no exec may touch

CLS = {dfft.SLAB_ZY_THEN_X: dfft.MPIcuFFT_Slab, dfft.SLAB_Z_THEN_YX: dfft.MPIcuFFT_Slab_Z_Then_YX, dfft.PENCIL: dfft.MPIcuFFT_Pencil}


def _plan(shape, prec, transform, batch, inplace, decomp=dfft.SLAB_ZY_THEN_X, scale=None):
    plan = CLS[decomp](dfft.Configurations(), dfft.Comm(), precision="double" if prec == dfft.F64 else "float",
                       transform="c2c" if transform == dfft.C2C else "r2c")
    plan.initFFT(dfft.GlobalSize(*shape), dfft.Partition(1, 1), True, batch, inplace)
    if scale is not None:
        plan.setScale(*scale)
    return plan


def _exec(plan, transform, inverse, out, in_, d):
    if transform == dfft.C2C:
        return plan.execC2C(out, in_, dfft.INVERSE if inverse else dfft.FORWARD, d)
    return plan.execC2R(out, in_, d) if inverse else plan.execR2C(out, in_, d)


def _refusal(plan, transform, inverse, out, in_, d):
    """the error code of an exec that must fail (0 if it did not); the exception is not kept, so no traceback holds this
    test's frames and buffers in a reference cycle"""
    try:
        _exec(plan, transform, inverse, out, in_, d)
    except DfftError as err:
        return err.code
    return 0


@pytest.fixture(autouse=True, scope="module")
def _release_buffers():
    """This module's buffers are tens of GiB: after its last test, collect whatever Python still holds in reference
    cycles and hand the cached device memory back, before the next module runs."""
    yield
    import gc

    import torch

    gc.collect()
    if torch.cuda.is_initialized():
        torch.cuda.empty_cache()


def compare(shape, prec, transform=dfft.C2C, batch=1, d=3, decomp=dfft.SLAB_ZY_THEN_X, scale=None):
    """forward then inverse, in place against out of place on the same input; bit-identical outputs, untouched canary"""
    import torch

    f64 = prec == dfft.F64
    rdt, cdt = (torch.float64, torch.complex128) if f64 else (torch.float32, torch.complex64)
    rs, cs = (8, 16) if f64 else (4, 8)
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    nzc = nz if c2c else nz // 2 + 1
    oop = _plan(shape, prec, transform, batch, False, decomp, scale)
    ip = _plan(shape, prec, transform, batch, True, decomp, scale)
    assert ip.isInPlace() and not oop.isInPlace()
    assert ip.getWorkSizeDevice() * 2 == oop.getWorkSizeDevice()
    dom = ip.getDomainSize()
    assert dom == oop.getDomainSize()
    osz = oop.getPartialSize(d)
    nout = osz[0] * osz[1] * osz[2]
    g = torch.Generator(device="cuda").manual_seed(17 + d)
    if c2c:
        x = torch.complex(torch.rand((batch, nx, ny, nz), generator=g, device="cuda", dtype=rdt),
                          torch.rand((batch, nx, ny, nz), generator=g, device="cuda", dtype=rdt)) - (0.5 + 0.5j)
    else:
        x = torch.rand((batch, nx, ny, nz), generator=g, device="cuda", dtype=rdt) - 0.5
    raw = torch.empty(batch * dom + CANARY, dtype=torch.uint8, device="cuda")
    raw[batch * dom:] = 0xA5
    base = raw.data_ptr()

    def field(f, nbytes, dtype):  # the first nbytes of field f of the buffer, as dtype
        return raw[f * dom:f * dom + nbytes].view(dtype)

    def load_real_side(src):  # C2C: the plain layout; R2C: padded rows of Nzc complex units
        for f in range(batch):
            if c2c:
                field(f, nx * ny * nz * cs, cdt).copy_(src[f].reshape(-1))
            else:
                field(f, nx * ny * nzc * cs, rdt).view(nx * ny, 2 * nzc)[:, :nz].copy_(src[f].reshape(nx * ny, nz))

    def real_side(f):
        if c2c:
            return field(f, nx * ny * nz * cs, cdt).view(nx, ny, nz)
        return field(f, nx * ny * nzc * cs, rdt).view(nx * ny, 2 * nzc)[:, :nz].reshape(nx, ny, nz)

    # forward
    spec = torch.empty((batch, nout), dtype=cdt, device="cuda")
    _exec(oop, transform, 0, spec, x, d)
    load_real_side(x)
    _exec(ip, transform, 0, base, base, d)
    torch.cuda.synchronize()
    for f in range(batch):
        assert torch.equal(field(f, nout * cs, cdt), spec[f]), f"forward field {f}: max |diff| {float((field(f, nout * cs, cdt) - spec[f]).abs().max())}"
    # inverse of the out-of-place spectrum
    back = torch.empty_like(x)
    _exec(oop, transform, 1, back, spec, d)
    for f in range(batch):
        field(f, nout * cs, cdt).copy_(spec[f])
    _exec(ip, transform, 1, base, base, d)
    torch.cuda.synchronize()
    for f in range(batch):
        assert torch.equal(real_side(f), back[f]), f"inverse field {f}: max |diff| {float((real_side(f) - back[f]).abs().max())}"
    assert bool((raw[batch * dom:] == 0xA5).all()), "an exec wrote beyond the buffer"
    # out != in is refused, on both directions and on the partial calls
    other = torch.empty(batch * dom, dtype=torch.uint8, device="cuda")
    for inverse in (0, 1):
        assert _refusal(ip, transform, inverse, other.data_ptr(), base, d) == -1
    ip.destroy()
    oop.destroy()
    del raw, other, x, spec, back
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("shape,prec,transform,batch", [
    ((512, 512, 512), dfft.F64, dfft.C2C, 1),     # fused z + y stage, both directions (in place: no discard in the inverse)
    ((1024, 256, 256), dfft.F64, dfft.C2C, 1),    # TMA x pass
    ((256, 256, 256), dfft.F32, dfft.C2C, 1),
    ((256, 256, 256), dfft.F64, dfft.R2C, 1),     # padded real rows
    ((256, 256, 256), dfft.F32, dfft.R2C, 1),
    ((96, 96, 96), dfft.F64, dfft.C2C, 1),        # Bluestein
    ((100, 120, 90), dfft.F64, dfft.C2C, 1),
    ((64, 64, 64), dfft.F64, dfft.C2C, 8),        # one-launch batched stage
    ((128, 128, 128), dfft.F64, dfft.C2C, 3),     # per field
    ((64, 32, 128), dfft.F64, dfft.R2C, 3),
])
def test_inplace_matches_out_of_place(shape, prec, transform, batch):
    compare(shape, prec, transform, batch)


@pytest.mark.gpu
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("transform", [dfft.C2C, dfft.R2C])
def test_inplace_partial(d, transform):
    compare((64, 128, 256), dfft.F64, transform, 1, d, dfft.PENCIL)
    compare((32, 64, 128), dfft.F32, transform, 2, d, dfft.PENCIL)


@pytest.mark.gpu
@pytest.mark.parametrize("decomp", [dfft.SLAB_Z_THEN_YX, dfft.PENCIL])
@pytest.mark.parametrize("transform", [dfft.C2C, dfft.R2C])
def test_inplace_other_decompositions(decomp, transform):
    compare((128, 64, 256), dfft.F64, transform, 1, 3, decomp)


@pytest.mark.gpu
def test_inplace_scale():
    n = 256 ** 3
    compare((256, 256, 256), dfft.F64, dfft.C2C, 1, scale=(1.0, 1.0 / n))
    compare((512, 512, 512), dfft.F64, dfft.C2C, 1, scale=(1.0, 1.0 / 512 ** 3))  # the scaled twin of the fused stage
    compare((256, 256, 256), dfft.F32, dfft.R2C, 1, scale=(1.0 / n, 1.0))
    compare((64, 64, 64), dfft.F64, dfft.C2C, 8, scale=(0.5, 1.0 / 64 ** 3))


@pytest.mark.gpu
def test_graph_replay_matches_eager():
    """one-rank in-place execs captured into a CUDA graph (forward then inverse) replay bit-identically to eager execs"""
    import torch

    for shape, batch in (((512, 512, 512), 1), ((64, 64, 64), 8), ((96, 96, 96), 1)):
        plan = _plan(shape, dfft.F64, dfft.C2C, batch, True)
        g = torch.Generator(device="cuda").manual_seed(3)
        x = torch.complex(torch.rand((batch,) + shape, generator=g, device="cuda", dtype=torch.float64),
                          torch.rand((batch,) + shape, generator=g, device="cuda", dtype=torch.float64))
        buf = x.clone()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            plan.execC2C(buf, buf, dfft.FORWARD, stream=s)
            plan.execC2C(buf, buf, dfft.INVERSE, stream=s)
        s.synchronize()
        eager = buf.clone()
        graph = torch.cuda.CUDAGraph()
        buf.copy_(x)
        torch.cuda.synchronize()
        with torch.cuda.graph(graph, stream=s):
            plan.execC2C(buf, buf, dfft.FORWARD, stream=s)
            plan.execC2C(buf, buf, dfft.INVERSE, stream=s)
        for _ in range(2):
            buf.copy_(x)
            graph.replay()
            torch.cuda.synchronize()
            plan.wait()
            assert torch.equal(buf, eager)
        del graph
        plan.destroy()
        del x, buf, eager
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_cpp_shim_inplace(tmp_path):
    """tests/cpp/inplace_shim_test.cpp: MPIcuFFT_Slab<double>::initFFT(gs, partition, allocate, batch, inplace) against the
    out-of-place plan, memcmp"""
    exe = str(tmp_path / "inplace_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include", os.path.join(HERE, "cpp", "inplace_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


@pytest.mark.gpu
def test_capacity_2048x1024x1024_complex_double():
    """32 GiB of data and a 32 GiB work area: 64 GiB in place instead of 128 GiB out of place.  Forward: DC term and
    Parseval against sums taken while the input was generated; inverse with scale 1/N: the input, checked chunk by chunk
    against the seeded input generated again (the input is not kept)."""
    import torch

    shape = (2048, 1024, 1024)
    N = shape[0] * shape[1] * shape[2]
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="c2c")
    plan.initFFT(dfft.GlobalSize(*shape), None, False, 1, True)  # no work area yet: size the need first
    field = N * 16
    assert plan.getDomainSize() == field and plan.getWorkSizeDevice() == field
    free, _ = torch.cuda.mem_get_info()
    if free < 2 * field + (6 << 30):
        plan.destroy()
        pytest.skip(f"needs {2 * field + (6 << 30)} free bytes on the device, {free} are free")
    work = torch.empty(field, dtype=torch.uint8, device="cuda")
    plan.setWorkArea(work)
    buf = torch.empty((shape[0], shape[1] * shape[2]), dtype=torch.complex128, device="cuda")
    CH = 64  # x planes per chunk: 1 GiB

    def chunk(c):
        g = torch.Generator(device="cuda").manual_seed(1000 + c)
        re = torch.rand((CH, shape[1] * shape[2]), generator=g, device="cuda", dtype=torch.float64) - 0.5
        im = torch.rand((CH, shape[1] * shape[2]), generator=g, device="cuda", dtype=torch.float64) - 0.5
        return torch.complex(re, im)

    total = torch.zeros((), dtype=torch.complex128, device="cuda")
    energy = torch.zeros((), dtype=torch.float64, device="cuda")
    for c in range(shape[0] // CH):
        v = chunk(c)
        total += v.sum()
        energy += (v.real ** 2 + v.imag ** 2).sum()
        buf[c * CH:(c + 1) * CH] = v
        del v
    plan.setScale(1.0, 1.0 / N)
    plan.execC2C(buf, buf, dfft.FORWARD)
    dc = complex(buf[0, 0].item())
    spec_energy = torch.zeros((), dtype=torch.float64, device="cuda")
    for c in range(shape[0] // CH):
        v = buf[c * CH:(c + 1) * CH]
        spec_energy += (v.real ** 2 + v.imag ** 2).sum()
    t, e, se = complex(total.item()), float(energy.item()), float(spec_energy.item())
    assert abs(dc - t) <= 1e-9 * (abs(t) + e ** 0.5), (dc, t)
    assert abs(se / N - e) <= 1e-10 * e, (se / N, e)
    plan.execC2C(buf, buf, dfft.INVERSE)
    worst = 0.0
    for c in range(shape[0] // CH):
        v = chunk(c)
        worst = max(worst, float((buf[c * CH:(c + 1) * CH] - v).abs().max()))
        del v
    assert worst < 1e-12, worst
    plan.destroy()
    del buf, work
    torch.cuda.empty_cache()
