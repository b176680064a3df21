"""Capture of one-rank plans into CUDA graphs: the `_async` execs recorded with torch.cuda.graph (and through the C ABI
with the raw runtime calls), replayed on fresh input, against eager execs of the same plan on the same input.  The same
kernels run on the same data, so every comparison is bit for bit.  Also the fused z + y stage's launch sequence on the
host (zy_launch_of), which is what makes its replays valid."""
import os
import subprocess
import tempfile

import pytest

import distributedfft_b200 as dfft
from distributedfft_b200._lib import DfftError

HERE = os.path.dirname(os.path.abspath(__file__))
DFFT_ERR_STATE = -4  # include/dfft.h


def test_fused_launch_sequence():
    """The fused kernel's (epoch, ticket) derived from the counter alone equals the host bookkeeping it replaces, over
    several launches drawing from one counter that is never reset."""
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "zy_launch_test")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "zy_launch_test.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0 and "fails=0" in r.stdout, r.stdout[-2000:]


# ---- GPU ------------------------------------------------------------------------------------------------------------
PLANS = {
    # name: (class, precision, transform, shape, partition, launches of the eager forward exec or None)
    "slab_c2c_fused_f64": (dfft.MPIcuFFT_Slab, dfft.F64, dfft.C2C, (64, 512, 512), None, 2),
    "slab_c2c_fused_f32": (dfft.MPIcuFFT_Slab, dfft.F32, dfft.C2C, (1024, 256, 256), None, 2),
    "slab_c2c_f64": (dfft.MPIcuFFT_Slab, dfft.F64, dfft.C2C, (128, 128, 128), None, None),
    "slab_r2c_f64": (dfft.MPIcuFFT_Slab, dfft.F64, dfft.R2C, (128, 128, 128), None, None),
    "z_then_yx_c2c_f32": (dfft.MPIcuFFT_Slab_Z_Then_YX, dfft.F32, dfft.C2C, (128, 128, 128), None, None),
    "pencil_r2c_f64": (dfft.MPIcuFFT_Pencil, dfft.F64, dfft.R2C, (128, 128, 128), (1, 1), None),
}


class Case:
    """A plan with its buffers: x -> out (forward), out -> back (inverse), all on torch's current stream."""

    def __init__(self, name):
        import torch

        cls, prec, transform, shape, part, self.launches = PLANS[name]
        self.c2c = transform == dfft.C2C
        self.f64 = prec == dfft.F64
        self.plan = cls(dfft.Configurations(), dfft.Comm(), precision="double" if self.f64 else "float",
                        transform="c2c" if self.c2c else "r2c")
        self.plan.initFFT(dfft.GlobalSize(*shape), dfft.Pencil_Partition(*part) if part else None, True)
        isz, osz = self.plan.getInSize(), self.plan.getOutSize()
        self.n_out = osz[0] * osz[1] * osz[2]
        self.rdt = torch.float64 if self.f64 else torch.float32
        cdt = torch.complex128 if self.f64 else torch.complex64
        n_in = isz[0] * isz[1] * isz[2]
        self.x = torch.empty(n_in, dtype=cdt if self.c2c else self.rdt, device="cuda")
        self.out = torch.empty(self.plan.getDomainSize() // (16 if self.f64 else 8), dtype=cdt, device="cuda")
        self.back = torch.empty_like(self.x)

    def refill(self, seed):
        import torch

        g = torch.Generator(device="cuda").manual_seed(seed)
        n = self.x.numel()
        if self.c2c:
            self.x.copy_(torch.complex(torch.rand(n, generator=g, device="cuda", dtype=self.rdt), torch.rand(n, generator=g, device="cuda", dtype=self.rdt)))
        else:
            self.x.copy_(torch.rand(n, generator=g, device="cuda", dtype=self.rdt))

    def fwd(self):
        import torch

        s = torch.cuda.current_stream()
        if self.c2c:
            self.plan.execC2C(self.out, self.x, dfft.FORWARD, stream=s)
        else:
            self.plan.execR2C(self.out, self.x, stream=s)

    def inv(self):
        import torch

        s = torch.cuda.current_stream()
        if self.c2c:
            self.plan.execC2C(self.back, self.out, dfft.INVERSE, stream=s)
        else:
            self.plan.execC2R(self.back, self.out, stream=s)

    def spectrum(self):
        return self.out[:self.n_out].clone()

    def capture(self, *fns):
        import torch

        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for fn in fns:
                fn()
        return g

    def destroy(self):
        import torch

        self.plan.destroy()
        del self.x, self.out, self.back
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(PLANS))
def test_replay_matches_eager(name):
    """Forward and inverse each captured after one eager exec, replayed on three fresh inputs; eager execs and replays
    alternating on one plan; one graph holding forward then inverse against the eager round trip."""
    import torch

    c = Case(name)
    c.refill(0)
    c.fwd()
    if c.launches is not None:
        assert c.plan.lastLaunchCount() == c.launches
    c.inv()
    c.plan.wait()
    gf = c.capture(c.fwd)
    gi = c.capture(c.inv)
    for seed in (1, 2, 3):
        c.refill(seed)
        gf.replay()
        got = c.spectrum()
        c.fwd()
        assert torch.equal(got, c.spectrum()), f"forward replay {seed}"
        gi.replay()
        got = c.back.clone()
        c.fwd()  # the spectrum again, whatever the inverse did to its input
        c.inv()
        assert torch.equal(got, c.back), f"inverse replay {seed}"
    # eager, replay, eager, replay on the same input
    c.refill(4)
    results = []
    for run in (c.fwd, gf.replay, c.fwd, gf.replay):
        c.out.zero_()
        run()
        results.append(c.spectrum())
    assert all(torch.equal(results[0], r) for r in results[1:])
    # forward then inverse in one graph
    grt = c.capture(c.fwd, c.inv)
    c.refill(5)
    c.fwd()
    c.inv()
    ref_out, ref_back = c.spectrum(), c.back.clone()
    c.out.zero_()
    c.back.zero_()
    grt.replay()
    assert torch.equal(c.spectrum(), ref_out) and torch.equal(c.back, ref_back)
    torch.cuda.synchronize()
    assert c.plan.wait() == 0
    del gf, gi, grt
    c.destroy()


@pytest.mark.gpu
@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_capture_before_eager_exec_is_refused():
    """The first exec of a direction sets up what a capture cannot: the capture is refused with DFFT_ERR_STATE, nothing
    is recorded, and the plan works eagerly afterwards.  A warmed-up forward does not admit the inverse."""
    import torch

    c = Case("slab_c2c_f64")
    c.refill(0)
    with pytest.raises(DfftError) as ei:
        c.capture(c.fwd)
    assert ei.value.code == DFFT_ERR_STATE
    c.fwd()
    c.plan.wait()
    with pytest.raises(DfftError) as ei:
        c.capture(c.inv)
    assert ei.value.code == DFFT_ERR_STATE
    ref = c.spectrum()
    g = c.capture(c.fwd)
    c.out.zero_()
    g.replay()
    assert torch.equal(c.spectrum(), ref)
    torch.cuda.synchronize()
    assert c.plan.wait() == 0
    del g
    c.destroy()


@pytest.mark.gpu
@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")
def test_replay_leaves_timer_and_launch_count():
    """With the phase timer on, replays record no events: step labels, step count and launch count stay those of the
    last eager exec."""
    import torch

    c = Case("slab_c2c_fused_f64")
    c.refill(0)
    c.plan.enableTimer(True)
    c.fwd()
    c.plan.wait()
    labels = [lab for lab, _ in c.plan.stepTimes()]
    launches = c.plan.lastLaunchCount()
    assert labels and launches == 2
    with pytest.raises(DfftError):
        c.capture(c.inv)  # refused: the inverse has not run eagerly
    g = c.capture(c.fwd)
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert [lab for lab, _ in c.plan.stepTimes()] == labels
    assert c.plan.lastLaunchCount() == launches
    assert c.plan.wait() == 0
    c.plan.enableTimer(False)
    del g
    c.destroy()


@pytest.mark.gpu
def test_cpp_graph_capture(tmp_path):
    """tests/cpp/graph_capture_test.cu: the same through the C ABI with cudaStreamBeginCapture / cudaGraphInstantiate /
    cudaGraphLaunch, compared with memcmp against eager output."""
    root = os.path.dirname(HERE)
    exe = str(tmp_path / "graph_capture_test")
    libdir = os.path.join(root, "distributedfft_b200")
    subprocess.run(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I" + os.path.join(root, "include"),
                    os.path.join(HERE, "cpp", "graph_capture_test.cu"), "-o", exe, "-L" + libdir, "-ldfft", "-Xlinker", "-rpath," + libdir],
                   check=True)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "PASSED" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
