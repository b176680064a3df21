"""Output scale on one GPU: a scaled exec stores exactly the unscaled output of the same plan times the scale, computed by
torch in the plan's dtype, bit for bit — for every kernel that has a scaled twin, in both directions, f32 and f64.  Also
the launch count and step list, the input and a canary after the last field, normalised round trips, CUDA graphs, the
return to (1, 1), and the C++ shim's setScale."""
import math
import os
import subprocess

import pytest

import distributedfft_b200 as dfft
from distributedfft_b200._lib import DfftError

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DFFT_ERR_STATE = -4
CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}

# name: (class, shape, transform, batch, d); every case runs f32 and f64 unless the name ends in _f64
CASES = {
    "slab_64_c2c": ("slab", (64, 64, 64), "c2c", 1, 3),                # three passes
    "slab_256_c2c_fused": ("slab", (256, 256, 256), "c2c", 1, 3),      # fused z + y stage
    "slab_512_c2c_fused_f64": ("slab", (512, 512, 512), "c2c", 1, 3),
    "slab_1024x64x64_f64": ("slab", (1024, 64, 64), "c2c", 1, 3),      # x pass of 1024 points: TMA-fed
    "slab_r2c": ("slab", (64, 32, 128), "r2c", 1, 3),                  # C2R final z pass
    "zyx_c2c": ("zyx", (32, 64, 128), "c2c", 1, 3),
    "zyx_r2c": ("zyx", (32, 64, 128), "r2c", 1, 3),
    "pencil_r2c_d1": ("pencil", (32, 64, 128), "r2c", 1, 1),            # R2C z pass is final
    "pencil_r2c_d2": ("pencil", (32, 64, 128), "r2c", 1, 2),
    "pencil_c2c_d1": ("pencil", (32, 64, 128), "c2c", 1, 1),
    "pencil_c2c_d2": ("pencil", (32, 64, 128), "c2c", 1, 2),
    "batch_32x4": ("slab", (32, 32, 32), "c2c", 4, 3),                 # one-launch batched stage
    "batch_64x4": ("slab", (64, 64, 64), "c2c", 4, 3),
    "batch_128x2": ("slab", (128, 128, 128), "c2c", 2, 3),             # per-field batched path
}
PARAMS = [(name, f64) for name in CASES for f64 in ((True,) if name.endswith("_f64") else (True, False))]


def transformed_points(shape, d):
    nx, ny, nz = shape
    return nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1)


class Case:
    def __init__(self, name, f64):
        import torch

        kind, self.shape, self.transform, self.batch, self.d = CASES[name]
        self.c2c = self.transform == "c2c"
        self.f64 = f64
        self.plan = CLASSES[kind](dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform=self.transform)
        self.plan.initFFT(dfft.GlobalSize(*self.shape), dfft.Partition(1, 1) if kind == "pencil" else None, True, batch=self.batch)
        self.rdt = torch.float64 if f64 else torch.float32
        self.cdt = torch.complex128 if f64 else torch.complex64
        isz = self.plan.getInSize()
        osz = self.plan.getPartialSize(self.d)
        self.in_shape, self.out_shape = tuple(isz), tuple(osz)
        self.n = transformed_points(self.shape, self.d)

    def buffers(self, inverse, seed=5):
        """input of the direction (a valid half spectrum for C2R) and an output with one canary field after the last"""
        import torch

        g = torch.Generator(device="cuda").manual_seed(seed)
        rnd = lambda shape: torch.rand(shape, generator=g, device="cuda", dtype=self.rdt) * 2 - 1
        real = rnd((self.batch,) + self.in_shape)
        x = real if not self.c2c else torch.complex(real, rnd(real.shape))
        if inverse:
            spec = torch.empty((self.batch,) + self.out_shape, dtype=self.cdt, device="cuda")
            self.run(spec, x, 0)  # at the plan's current forward scale (1 when buffers are made)
            x = spec
        out_dt = self.cdt if (not inverse or self.c2c) else self.rdt
        out_shape = self.in_shape if inverse else self.out_shape
        out = torch.full((self.batch + 1,) + out_shape, 7.0, dtype=out_dt, device="cuda")
        return x, out

    def run(self, out, x, inverse, stream=None):
        if self.c2c:
            self.plan.execC2C(out, x, dfft.INVERSE if inverse else dfft.FORWARD, d=self.d, stream=stream)
        elif inverse:
            self.plan.execC2R(out, x, d=self.d, stream=stream)
        else:
            self.plan.execR2C(out, x, d=self.d, stream=stream)


def bits(t):
    import torch

    r = torch.view_as_real(t) if t.is_complex() else t
    return r.contiguous().view(torch.int64 if r.dtype == torch.float64 else torch.int32)


def times(t, s):
    """t * s as torch computes it in t's dtype: a real multiply of every real and imaginary part"""
    import torch

    r = torch.view_as_real(t) if t.is_complex() else t
    return r * torch.tensor(s, dtype=r.dtype, device=r.device)


@pytest.mark.gpu
@pytest.mark.parametrize("name,f64", PARAMS)
def test_scaled_equals_unscaled_times_s(name, f64, monkeypatch):
    import torch

    monkeypatch.delenv("DFFT_TMA", raising=False)
    envs = [{}]
    if name.startswith("slab_1024x64x64"):
        envs = [{}, {"DFFT_TMA": "0"}, {"DFFT_BULK_STORE": "1"}]
    for env in envs:
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        c = Case(name, f64)
        c.plan.enableTimer(True)
        for inverse in (0, 1):
            x, out = c.buffers(inverse)
            x_copy = x.clone()
            c.run(out[:c.batch], x, inverse)
            torch.cuda.synchronize()
            ref = out[:c.batch].clone()
            launches, labels = c.plan.lastLaunchCount(), [l for l, _ in c.plan.stepTimes()]
            for s in (1.0 / c.n, 1.0 / math.sqrt(c.n), 0.3, -2.5):
                c.plan.setScale(*((1.0, s) if inverse else (s, 1.0)))
                assert c.plan.getScale() == ((1.0, s) if inverse else (s, 1.0))
                out[:c.batch].fill_(7.0)
                c.run(out[:c.batch], x, inverse)
                torch.cuda.synchronize()
                sf = s if f64 else float(torch.tensor(s, dtype=torch.float32))
                assert torch.equal(bits(out[:c.batch]), bits(times(ref, sf))), (name, env, inverse, s)
                assert torch.equal(bits(x), bits(x_copy)), "the input was modified"
                assert bool((out[c.batch] == 7.0).all()), "the canary after the last field was overwritten"
                assert c.plan.lastLaunchCount() == launches
                assert [l for l, _ in c.plan.stepTimes()] == labels
            # back to (1, 1): bit-identical to the unscaled output
            c.plan.setScale(1.0, 1.0)
            c.run(out[:c.batch], x, inverse)
            torch.cuda.synchronize()
            assert torch.equal(bits(out[:c.batch]), bits(ref))
        c.plan.destroy()
        for k in env:
            monkeypatch.delenv(k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["slab_64_c2c", "slab_256_c2c_fused", "slab_r2c", "zyx_r2c", "pencil_c2c_d2", "batch_64x4", "batch_128x2"])
@pytest.mark.parametrize("f64", [True, False])
def test_normalised_round_trip(name, f64):
    """setScale(1, 1/N): inverse(forward(x)) is x, with no scaling by the caller"""
    import torch

    c = Case(name, f64)
    c.plan.setScale(1.0, 1.0 / c.n)
    x, spec = c.buffers(0)
    c.run(spec[:c.batch], x, 0)
    back = torch.empty_like(x)
    c.run(back, spec[:c.batch], 1)
    torch.cuda.synchronize()
    err = (torch.linalg.vector_norm(back - x) / torch.linalg.vector_norm(x)).item()
    assert err <= (1e-12 if f64 else 1e-6), err
    c.plan.destroy()


@pytest.mark.gpu
@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
@pytest.mark.parametrize("name,f64", [("slab_64_c2c", True), ("slab_256_c2c_fused", True), ("slab_r2c", False), ("batch_64x4", True)])
def test_graph_replay_keeps_its_scale(name, f64):
    """a replay equals the eager scaled exec; a graph keeps the scale it was captured with after setScale; capturing
    right after setScale is refused until the direction has run eagerly again"""
    import torch

    c = Case(name, f64)

    def capture(out, x, inverse):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c.run(out, x, inverse, stream=torch.cuda.current_stream())
        return g

    for inverse in (0, 1):
        scale = (1.0, 0.3) if inverse else (0.3, 1.0)
        x, out = c.buffers(inverse)
        c.plan.setScale(*scale)
        c.run(out[:c.batch], x, inverse, stream=torch.cuda.current_stream())  # eager: sets up the scaled kernels
        torch.cuda.synchronize()
        eager = out[:c.batch].clone()
        g = capture(out[:c.batch], x, inverse)
        out.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(out[:c.batch]), bits(eager))
        c.plan.setScale(1.0, 1.0)
        with pytest.raises(DfftError) as e:
            capture(out[:c.batch], x, inverse)
        assert e.value.code == DFFT_ERR_STATE
        out.fill_(0)
        g.replay()  # the old graph still applies 0.3
        torch.cuda.synchronize()
        assert torch.equal(bits(out[:c.batch]), bits(eager))
        c.run(out[:c.batch], x, inverse, stream=torch.cuda.current_stream())  # eager at (1, 1): capturable again
        torch.cuda.synchronize()
        plain = out[:c.batch].clone()
        g1 = capture(out[:c.batch], x, inverse)
        out.fill_(0)
        g1.replay()
        torch.cuda.synchronize()
        assert torch.equal(bits(out[:c.batch]), bits(plain))
        del g, g1
    c.plan.destroy()


@pytest.mark.gpu
def test_cpp_shim_set_scale(tmp_path):
    """tests/cpp/scale_shim_test.cpp: MPIcuFFT_Slab<double> with setScale(1, 1/N) round-trips R2C -> C2R to the input"""
    exe = str(tmp_path / "scale_shim_test")
    libdir = os.path.join(ROOT, "distributedfft_b200")
    subprocess.run(["g++", "-std=c++17", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include", os.path.join(HERE, "cpp", "scale_shim_test.cpp"),
                    "-o", exe, "-L" + libdir, "-ldfft", "-L/usr/local/cuda/lib64", "-lcudart", "-Wl,-rpath," + libdir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout + r.stderr
