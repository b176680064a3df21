"""Batched plans on one GPU: every field of a batched exec equals the unbatched plan's output on that field bit for bit
(the one-launch stage and the per-field path), matches cufftPlanMany, leaves the input and the memory after the last
field untouched, and replays bit-identically from a CUDA graph; the C++ shim's batched initFFT."""
import ctypes as C
import os
import subprocess

import pytest

import distributedfft_b200 as dfft

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}


@pytest.fixture(scope="module")
def cufft_many(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cufft") / "libcufft_many_ref.so")
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC",
                    os.path.join(ROOT, "tools", "cufft_many_ref.cu"), "-lcufft", "-o", so], check=True)
    lib = C.CDLL(so)
    lib.cufft_ref_3d_many.restype = C.c_int
    lib.cufft_ref_3d_many.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_int]
    return lib


def make_plan(kind, n, f64, transform, batch):
    plan = CLASSES[kind](dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform=transform)
    part = dfft.Partition(1, 1) if kind == "pencil" else None
    plan.initFFT(dfft.GlobalSize(*n), part, True, batch=batch)
    assert plan.getBatch() == batch
    return plan


def rand(shape, f64, complex_, seed):
    import torch
    rdt = torch.float64 if f64 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(seed)
    re = torch.rand(shape, generator=g, device="cuda", dtype=rdt) * 255
    if not complex_:
        return re
    return torch.complex(re, torch.rand(shape, generator=g, device="cuda", dtype=rdt) * 255)


def exec_(plan, transform, inverse, out, x, stream=None):
    if transform == "c2c":
        plan.execC2C(out, x, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)
    elif inverse:
        plan.execC2R(out, x, stream=stream)
    else:
        plan.execR2C(out, x, stream=stream)


def check_case(kind, n, f64, transform, inverse, batch, launches_per_exec):
    """batched exec vs the unbatched plan per field: bit-identical, input intact, canary after the last field untouched"""
    import torch
    c2c = transform == "c2c"
    nzc = n[2] if c2c else n[2] // 2 + 1
    real_shape, cplx_shape = tuple(n), (n[0], n[1], nzc)
    in_shape, out_shape = (cplx_shape, real_shape) if inverse else (real_shape, cplx_shape)
    in_complex, out_complex = (True, c2c) if inverse else (c2c, True)
    x = rand((batch,) + in_shape, f64, in_complex, 7)
    if not c2c and inverse:  # a valid half spectrum: the forward transform of real fields
        pf = make_plan(kind, n, f64, transform, 1)
        src = rand((batch,) + real_shape, f64, False, 7)
        for f in range(batch):
            exec_(pf, transform, False, x[f], src[f])
        pf.destroy()
    x_copy = x.clone()
    cdt = (torch.complex128 if f64 else torch.complex64) if out_complex else (torch.float64 if f64 else torch.float32)
    out = torch.full((batch + 1,) + out_shape, 3.0, device="cuda", dtype=cdt)  # field `batch`: canary
    pb = make_plan(kind, n, f64, transform, batch)
    exec_(pb, transform, inverse, out[:batch], x)
    assert pb.lastLaunchCount() == launches_per_exec
    p1 = make_plan(kind, n, f64, transform, 1)
    want = torch.empty((batch,) + out_shape, device="cuda", dtype=cdt)
    for f in range(batch):
        exec_(p1, transform, inverse, want[f], x_copy[f])
    torch.cuda.synchronize()
    assert torch.equal(x, x_copy), "the input was modified"
    assert bool((out[batch] == 3.0).all()), "memory after the last field was written"
    for f in range(batch):
        assert torch.equal(out[f], want[f]), f"field {f}: max |diff| {float((out[f] - want[f]).abs().max())}"
    pb.destroy()
    p1.destroy()
    return out[:batch], x


@pytest.mark.gpu
@pytest.mark.parametrize("n", [32, 64])
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("inverse", [0, 1])
def test_batched_stage_is_bit_identical(n, f64, inverse):
    check_case("slab", (n, n, n), f64, "c2c", inverse, 5, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,n,transform,inverse,batch,per_field", [
    ("slab", (128, 128, 128), "c2c", 0, 3, 3), ("slab", (128, 128, 128), "c2c", 1, 3, 3),
    ("slab", (128, 128, 128), "r2c", 0, 3, 3), ("slab", (128, 128, 128), "r2c", 1, 3, 3),
    ("zyx", (64, 32, 64), "c2c", 0, 3, 3), ("zyx", (64, 32, 64), "r2c", 1, 2, 3),
    ("pencil", (32, 32, 32), "c2c", 0, 4, 3), ("pencil", (32, 64, 32), "r2c", 1, 2, 3),
])
def test_per_field_path_is_bit_identical(kind, n, transform, inverse, batch, per_field):
    check_case(kind, n, True, transform, inverse, batch, batch * per_field)


@pytest.mark.gpu
@pytest.mark.parametrize("n,f64,batch", [(32, True, 6), (64, True, 4), (32, False, 6), (64, False, 4), (128, True, 2)])
def test_batched_vs_cufft_plan_many(cufft_many, n, f64, batch):
    import torch
    x = rand((batch, n, n, n), f64, True, 11)
    ref, back = torch.empty_like(x), torch.empty_like(x)
    plan = make_plan("slab", (n, n, n), f64, "c2c", batch)
    out = torch.empty_like(x)
    plan.execC2C(out, x, dfft.FORWARD)
    ms = C.c_float()
    assert cufft_many.cufft_ref_3d_many(1 if f64 else 0, 0, n, n, n, batch, ref.data_ptr(), x.data_ptr(), C.byref(ms), 1) == 0
    tol = 1e-10 if f64 else 1e-5
    rel = lambda a, b: float((a - b).abs().pow(2).sum().sqrt() / b.abs().pow(2).sum().sqrt())  # noqa: E731
    for f in range(batch):
        assert rel(out[f], ref[f]) < tol, f
    plan.execC2C(back, ref, dfft.INVERSE)
    assert cufft_many.cufft_ref_3d_many(1 if f64 else 0, 1, n, n, n, batch, out.data_ptr(), ref.data_ptr(), C.byref(ms), 1) == 0
    for f in range(batch):
        assert rel(back[f], out[f]) < tol, f
    plan.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("n,batch,launches", [(64, 4, 1), (32, 7, 1), (128, 2, 6)])
def test_batched_graph_replay(n, batch, launches):
    """captured batched execs (one launch, and the per-field path) replay bit-identically to eager ones, repeatedly"""
    import torch
    x = rand((batch, n, n, n), True, True, 3)
    plan = make_plan("slab", (n, n, n), True, "c2c", batch)
    out, back = torch.empty_like(x), torch.empty_like(x)
    s = torch.cuda.current_stream()
    plan.execC2C(out, x, dfft.FORWARD, stream=s)
    plan.execC2C(back, out, dfft.INVERSE, stream=s)
    plan.wait()
    assert plan.lastLaunchCount() == launches
    want_f, want_i = out.clone(), back.clone()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        plan.execC2C(out, x, dfft.FORWARD, stream=torch.cuda.current_stream())
        plan.execC2C(back, out, dfft.INVERSE, stream=torch.cuda.current_stream())
    for _ in range(3):
        out.zero_()
        back.zero_()
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, want_f) and torch.equal(back, want_i)
        plan.execC2C(out, x, dfft.FORWARD, stream=s)  # eager execs between replays share the counters
        plan.wait()
        assert torch.equal(out, want_f)
    del gr
    plan.destroy()


@pytest.mark.gpu
def test_cpp_shim_batched_init(tmp_path):
    """tests/cpp/batch_shim_test.cpp: MPIcuFFT_Slab<double>::initFFT(gs, partition, allocate, batch) against the unbatched
    plan per field, memcmp"""
    exe = str(tmp_path / "batch_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include", os.path.join(HERE, "cpp", "batch_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
