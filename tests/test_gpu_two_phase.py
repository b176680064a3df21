"""The persistent two-phase stages, exec after exec: the fused z + y stage (fft_zy_fused_kernel / fft_zy_fed_kernel) and the
batched small-field stage (fft_batch_small_kernel).

Both stages hand an intermediate from phase-A items to phase-B items of other CTAs through memory: the plan's work area for
the fused stage, the caller's `out` for the batched stage.  A phase-B item that reads too early, or a line discarded before
its last reader, returns whatever that memory held before.  When every exec repeats the same input, that is the previous
exec's intermediate, which is exactly right; so every exec here gets a new input, and the memory the intermediate passes
through is filled with NaN (all-ones bytes) before it:
  - fused plans are created without a work area and run on a caller-owned arena: the work bytes refilled with 0xFF before
    every eager exec, a guard of GUARD bytes on either side holding a fixed non-NaN pattern that must survive every exec;
  - batched plans get `out` filled with NaN before every exec;
  - consecutive execs never share an input or output buffer.
Every output is compared bit for bit with the standalone passes run on the same input (fused stage: fft1d_contig along z,
fft1d_strided along y, fft1d_general along x, in the plan's order; batched stage: the unbatched plan, field by field); a
scaled inverse with the unscaled composition times the scale, in the plan's dtype.  Each case asserts it ran the stage it
is meant to test: the launch count and the live plan's step labels (dfft_plan_describe), with the L2 size read from the
device as the plan reads it.  A few cases are also checked against a long-double reference (error_check of
test_gpu_schedule_replay), so that a wrong standalone pass cannot hide behind bit equality.  Measured on an H100 80GB HBM3
(700 W), in units of u sqrt(sum log2 L), rel-L2 / max over rms(ref): f64 0.81 / 4.07, f32 0.91 / 4.63 (bounds 3 / 30).  The
module's GPU tests take about 35 s there.

The CPU tests at the end pin, with geometry-only plans (which assume a 50 MiB L2), which of the sweep's shapes fuse, so
that the GPU tests' coverage cannot shrink silently, and replay the smallest fused shape with a Bluestein x pass."""
import json

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from test_schedule_emulation import P2P, SL, SYNC, run_case

F32, F64 = dfft.F32, dfft.F64
ESIZE = {F64: 16, F32: 8}
GUARD = 64 << 10  # bytes of guard before and after the work bytes of an arena (keeps the work area 64 KiB aligned)
GUARD_BYTE = 0x5A  # 0x5A5A5A5A / 0x5A5A...5A: finite in f32 and f64
DRY_L2 = 50 << 20  # the L2 geometry-only plans assume
FUSED_FWD = ["zy pass: z phase", "zy pass: y phase", "x pass"]
FUSED_INV = ["x pass", "yz pass: y phase", "yz pass: z phase"]
PLAIN_FWD = ["z pass", "y pass", "x pass"]
PLAIN_INV = ["x pass", "y pass", "z pass"]


# ---- which shapes run which stage (the plan's own rules, from the L2 size) ----------------------------------------------------
def fused_nx(role, n, prec, l2):
    """nx of a sweep role: "min" the smallest nx whose array exceeds the L2, "min+1", "pow2" (64; 128 for 256^2 f32 planes,
    where 64 planes fit the L2) and "100" (not a power of two; exactly the L2 for 256^2 f32 planes: not fused)"""
    smallest = l2 // (n * n * ESIZE[prec]) + 1
    return {"min": smallest, "min+1": smallest + 1, "pow2": 128 if (n, prec) == (256, F32) else 64, "100": 100}[role]


def is_fused(nx, n, prec, l2):
    """zy_fused() for one-rank slab C2C plans of Ny = Nz = n in {256, 512}: the blocked hand-over is 32 columns wide for
    these lengths, and the array must not fit the L2"""
    return nx * n * n * ESIZE[prec] > l2


def default_ahead(n, prec, l2, fields=False):
    """the look-ahead of fuse_zy (planes) or build_batch_small (fields, n^3 each)"""
    per = n * n * (n if fields else 1) * ESIZE[prec]
    return max(1, l2 // (3 * per) - 1)


def ahead_of(role, nx):
    """DFFT_ZY_AHEAD of a sweep role (None: the plan's default); nx - 1, nx and nx + 5 take the L >= n branch of
    ZyOrder::decode"""
    return {"1": 1, "2": 2, "default": None, "nx-1": nx - 1, "nx": nx, "nx+5": nx + 5}[role]


def labels(sc):
    return [s["label"] for s in sc["steps"]]


def expected_labels(fused, inverse, batch=1):
    if fused:
        return (FUSED_INV if inverse else FUSED_FWD) * batch
    return (PLAIN_INV if inverse else PLAIN_FWD) * batch


PRECS = [(512, F64), (512, F32), (256, F64), (256, F32)]
ROLES = ["min", "min+1", "pow2", "100"]
AHEADS = ["1", "2", "default", "nx-1", "nx", "nx+5"]
# the main sweep: every (planes, precision) with every nx role, the look-ahead rotating so that every look-ahead meets
# several nx roles and both plane sizes
SWEEP = [(n, prec, role, AHEADS[(4 * i + j) % len(AHEADS)]) for i, (n, prec) in enumerate(PRECS) for j, role in enumerate(ROLES)]
# batch 3 through the fused stage, out of place and in place, and single in-place fields
LAYOUTS = [(512, F64, "min", 3, False), (512, F64, "min", 3, True), (256, F32, "min", 3, True), (256, F64, "min", 1, True),
           (512, F32, "min+1", 1, True), (256, F32, "pow2", 3, False)]
BATCH_SIZES = lambda ahead: sorted({2, ahead, ahead + 1, 2 * ahead + 1, 17 if ahead != 17 else 19})  # noqa: E731


# ---- GPU helpers -------------------------------------------------------------------------------------------------------------
def device_l2():
    import torch

    return int(torch.cuda.get_device_properties(0).L2_cache_size)


def cdt(prec):
    import torch

    return torch.complex128 if prec == F64 else torch.complex64


def bits(t):
    import torch

    r = torch.view_as_real(t)
    return r.view(torch.int64 if r.dtype == torch.float64 else torch.int32)


def rand(shape, prec, seed):
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    rdt = torch.float64 if prec == F64 else torch.float32
    return torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt) * 2 - 1,
                         torch.rand(shape, generator=g, device="cuda", dtype=rdt) * 2 - 1)


def nan_(t):
    import torch

    torch.view_as_real(t).fill_(float("nan"))
    return t


def has_nan(t):
    import torch

    return bool(torch.isnan(torch.view_as_real(t)).any())


def times(t, s, prec):
    """t * s as torch computes it in t's dtype (f32 plans apply s rounded to float)"""
    import torch

    r = torch.view_as_real(t)
    sf = s if prec == F64 else float(np.float32(s))
    return torch.view_as_complex(r * torch.tensor(sf, dtype=r.dtype, device=r.device))


def live_schedule(plan, inverse):
    return json.loads(R.describe_raw(plan._h, inverse, 3))


class Arena:
    """a caller-owned work area with a guard on either side"""

    def __init__(self, plan):
        import torch

        self.work = plan.getWorkSizeDevice()
        assert self.work > 0
        self.buf = torch.empty(2 * GUARD + self.work, dtype=torch.uint8, device="cuda")
        self.buf[:GUARD].fill_(GUARD_BYTE)
        self.buf[GUARD + self.work:].fill_(GUARD_BYTE)
        self.poison()
        plan.setWorkArea(self.buf[GUARD:].data_ptr())
        assert plan.getWorkAreaDevice() == self.buf[GUARD:].data_ptr()

    def area(self):
        return self.buf[GUARD:GUARD + self.work]

    def poison(self):
        self.area().fill_(0xFF)  # NaN in f32 and f64

    def check_guards(self):
        assert bool((self.buf[:GUARD] == GUARD_BYTE).all()), "the guard before the work area was overwritten"
        assert bool((self.buf[GUARD + self.work:] == GUARD_BYTE).all()), "the guard after the work area was overwritten"

    def used(self):
        return not bool((self.area() == 0xFF).all())


def composed(prec, nx, n, direction, x):
    """the standalone passes in the fused plan's order on one field x [nx][n][n]: forward z, y, x; inverse x, y, z"""
    import torch

    s = torch.cuda.current_stream()
    a, b = torch.empty_like(x), torch.empty_like(x)
    if direction == dfft.FORWARD:
        dfft.fft1d_contig(prec, 0, direction, n, nx * n, a, n, x, n, s)
        dfft.fft1d_strided(prec, direction, nx, n, n, b, a, s)
        dfft.fft1d_general(prec, direction, nx, 1, 1, n * n, a, (0, 0, n * n), b, (0, 0, n * n), s)
    else:
        dfft.fft1d_general(prec, direction, nx, 1, 1, n * n, a, (0, 0, n * n), x, (0, 0, n * n), s)
        dfft.fft1d_strided(prec, direction, nx, n, n, b, a, s)
        dfft.fft1d_contig(prec, 0, direction, n, nx * n, a, n, b, n, s)
    return a


class FusedCase:
    """a slab C2C plan of nx x n x n on a poisoned caller-owned arena; `fused` is what the plan's rules give for this GPU"""

    def __init__(self, n, prec, nx, batch=1, inplace=False):
        self.n, self.prec, self.nx, self.batch, self.inplace = n, prec, nx, batch, inplace
        self.shape = (batch, nx, n, n) if batch > 1 else (nx, n, n)
        self.plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if prec == F64 else "float", transform="c2c")
        self.plan.initFFT(dfft.GlobalSize(nx, n, n), None, False, batch=batch, inplace=inplace)
        if inplace:
            assert self.plan.getDomainSize() == nx * n * n * ESIZE[prec]
        self.arena = Arena(self.plan)
        self.fused = is_fused(nx, n, prec, device_l2())
        self.launches = 2 * batch if self.fused else 3 * batch
        self.seed = 1000 * nx + n + 7 * prec + 13 * batch

    def check_stage(self, inverse):
        sc = live_schedule(self.plan, inverse)
        assert labels(sc) == expected_labels(self.fused, inverse, self.batch), labels(sc)
        x_pass = [s for s in sc["steps"] if s["label"] == "x pass"]
        assert len(x_pass) == self.batch
        # a non-power-of-two nx runs the Bluestein x pass (its step carries "n")
        assert all(s.get("n", 0) == (0 if self.nx & (self.nx - 1) == 0 else self.nx) for s in x_pass)

    def new_input(self):
        self.seed += 1
        return rand(self.shape, self.prec, self.seed)

    def want(self, x, direction, scale=1.0):
        import torch

        fields = x if self.batch > 1 else x.unsqueeze(0)
        ref = torch.stack([composed(self.prec, self.nx, self.n, direction, f) for f in fields])
        ref = ref if self.batch > 1 else ref[0]
        return ref if scale == 1.0 else times(ref, scale, self.prec)

    def run(self, out, x, direction, stream=None):
        self.plan.execC2C(out, x, direction, stream=stream)

    def check(self, got, want, what):
        import torch

        torch.cuda.synchronize()
        self.arena.check_guards()
        assert not has_nan(got), f"{what}: NaN in the output (an intermediate read before it was written, or discarded early)"
        if not torch.equal(bits(got), bits(want)):
            diff = (got != want).reshape(-1).nonzero()
            first = int(diff[0])
            raise AssertionError(f"{what}: {diff.numel()} elements differ, first at flat index {first} "
                                 f"(field/plane/row/col {np.unravel_index(first, got.shape)}), got {complex(got.reshape(-1)[first])} "
                                 f"want {complex(want.reshape(-1)[first])}")

    def destroy(self):
        self.plan.destroy()


def eager_sequence(c, direction, scale, execs, feeds, monkeypatch, tag):
    """`execs` eager execs of one direction, each on a new input, alternating two outputs (in place: a new buffer each)"""
    import torch

    outs = [nan_(torch.empty(c.shape, dtype=cdt(c.prec), device="cuda")) for _ in range(2)]
    for i in range(execs):
        feed = feeds[i % len(feeds)]
        if feed is not None:
            monkeypatch.setenv("DFFT_ZY_FEED", str(feed))  # read by the launcher at every exec
        x = c.new_input()
        want = c.want(x, direction, scale)
        c.arena.poison()
        if c.inplace:
            buf = x.clone()
            c.run(buf, buf, direction)
            got = buf
        else:
            got = nan_(outs[i % 2])
            x_copy = x.clone()
            c.run(got, x, direction)
        assert c.plan.lastLaunchCount() == c.launches
        c.check(got, want, f"{tag} exec {i} (DFFT_ZY_FEED={feed})")
        if not c.inplace:
            assert torch.equal(bits(x), bits(x_copy)), "the input was modified"
        if i == 0:
            assert c.arena.used(), "the exec left the whole work area NaN: it does not run on the caller's arena"


def run_directions(c, monkeypatch, execs, feeds):
    for direction, scale in ((dfft.FORWARD, 1.0), (dfft.INVERSE, 1.0), (dfft.INVERSE, 1.0 / 3)):
        inverse = 1 if direction == dfft.INVERSE else 0
        c.plan.setScale(1.0, scale)
        c.check_stage(inverse)
        eager_sequence(c, direction, scale, execs, feeds, monkeypatch, f"direction {direction} scale {scale}")
    c.plan.setScale(1.0, 1.0)


def feeds_of(prec):
    return (1, 0) if prec == F64 else (None,)


# ---- GPU: the fused z + y stage ----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n,prec,role,ahead", SWEEP)
def test_fused_exec_after_exec(n, prec, role, ahead, monkeypatch):
    """new input every exec, poisoned arena, forward / inverse / scaled inverse, both kernels in f64, every look-ahead"""
    import torch

    l2 = device_l2()
    nx = fused_nx(role, n, prec, l2)
    a = ahead_of(ahead, nx)
    monkeypatch.delenv("DFFT_ZY_AHEAD", raising=False)
    if a is not None:
        monkeypatch.setenv("DFFT_ZY_AHEAD", str(a))  # read when the schedule is built
    c = FusedCase(n, prec, nx)
    if role != "100":
        assert c.fused, (nx, n, prec, l2)
    run_directions(c, monkeypatch, 4 if prec == F64 else 3, feeds_of(prec))
    c.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("n,prec,role,batch,inplace", LAYOUTS)
def test_fused_batch_and_inplace(n, prec, role, batch, inplace, monkeypatch):
    """batches through the fused stage (one launch pair per field) and in-place plans, field by field against the
    standalone passes"""
    import torch

    monkeypatch.delenv("DFFT_ZY_AHEAD", raising=False)
    nx = fused_nx(role, n, prec, device_l2())
    c = FusedCase(n, prec, nx, batch, inplace)
    assert c.fused
    run_directions(c, monkeypatch, 3, feeds_of(prec))
    c.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("n,prec,role,inverse", [(512, F64, "min", 0), (256, F32, "min", 1), (256, F64, "pow2", 1), (512, F32, "100", 0)])
def test_fused_graph_replay_between_eager_execs(n, prec, role, inverse, monkeypatch):
    """a captured exec replayed between eager ones, each on a new input: the counters' epochs carry across both kinds of
    launch"""
    import torch

    monkeypatch.delenv("DFFT_ZY_AHEAD", raising=False)
    c = FusedCase(n, prec, fused_nx(role, n, prec, device_l2()))
    assert c.fused
    direction = dfft.INVERSE if inverse else dfft.FORWARD
    c.check_stage(inverse)
    s = torch.cuda.current_stream()
    cap_x = torch.empty(c.shape, dtype=cdt(prec), device="cuda")
    cap_out = torch.empty_like(cap_x)
    eager_out = [torch.empty_like(cap_x) for _ in range(2)]
    # the direction runs eagerly once before it can be captured
    x = c.new_input()
    c.arena.poison()
    c.run(nan_(eager_out[1]), x, direction, stream=s)
    c.check(eager_out[1], c.want(x, direction), "first eager exec")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        c.run(cap_out, cap_x, direction, stream=torch.cuda.current_stream())
    for i, kind in enumerate(["eager", "replay", "eager", "replay", "eager", "replay"]):
        x = c.new_input()
        want = c.want(x, direction)
        c.arena.poison()
        if kind == "replay":
            cap_x.copy_(x)
            nan_(cap_out)
            g.replay()
            got = cap_out
        else:
            got = nan_(eager_out[i % 2])
            c.run(got, x, direction, stream=s)
            assert c.plan.lastLaunchCount() == 2
        c.check(got, want, f"{kind} {i}")
    del g
    c.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("n,prec,role", [(512, F64, "min+1"), (256, F32, "min")])
def test_fused_back_to_back(n, prec, role, monkeypatch):
    """K async execs enqueued on one stream with no host sync between them, each with its own input and output, the
    arena re-poisoned in stream order before each"""
    import torch

    K = 4
    monkeypatch.delenv("DFFT_ZY_AHEAD", raising=False)
    c = FusedCase(n, prec, fused_nx(role, n, prec, device_l2()))
    assert c.fused
    for direction in (dfft.FORWARD, dfft.INVERSE):
        xs = [c.new_input() for _ in range(K)]
        outs = [nan_(torch.empty_like(xs[0])) for _ in range(K)]
        torch.cuda.synchronize()
        s = torch.cuda.current_stream()
        for k in range(K):
            c.arena.poison()
            c.run(outs[k], xs[k], direction, stream=s)
        for k in range(K):
            c.check(outs[k], c.want(xs[k], direction), f"direction {direction}, exec {k} of {K}")
    c.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_fused_beside_a_gemm(monkeypatch):
    """One fused exec started while a large GEMM runs on another stream, so the persistent kernel can begin with fewer
    resident CTAs than its grid: the wait in ticket_loop must still make progress.  A wrong claim there ends in DFFT_ERR_TIMEOUT
    after 60 s instead of a hang."""
    import torch

    monkeypatch.setenv("DFFT_RENDEZVOUS_TIMEOUT_S", "60")  # read at plan creation
    monkeypatch.delenv("DFFT_ZY_AHEAD", raising=False)
    monkeypatch.setenv("DFFT_ZY_FEED", "1")
    n, prec = 512, F64
    c = FusedCase(n, prec, 64)
    assert c.fused
    x = c.new_input()
    want = c.want(x, dfft.FORWARD)
    out = nan_(torch.empty_like(x))
    a = torch.rand((8192, 8192), device="cuda")
    b = torch.rand((8192, 8192), device="cuda")
    c.arena.poison()
    torch.cuda.synchronize()
    side, main = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(side):
        for _ in range(4):
            a = (a @ b) * (1.0 / 8192)
    c.run(out, x, dfft.FORWARD, stream=main)
    c.plan.wait()
    torch.cuda.synchronize()
    assert c.plan.lastLaunchCount() == 2
    c.check(out, want, "fused exec beside a GEMM")
    c.destroy()
    del a, b
    torch.cuda.empty_cache()


# ---- GPU: against a long-double reference --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("prec,nx,n", [(F64, 51, 256), (F32, 101, 256)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_fused_vs_long_double(prec, nx, n, inverse):
    """the smallest fused shape of 256^2 planes at 50 MiB of L2 (a Bluestein x pass) against np.fft in long double:
    rel-L2 <= 3 and max <= 30 in units of u sqrt(sum log2 L), the bounds of test_gpu_schedule_replay"""
    import torch
    from test_gpu_accuracy import spec
    from test_gpu_schedule_replay import error_check

    c = FusedCase(n, prec, nx)
    direction = dfft.INVERSE if inverse else dfft.FORWARD
    rng = np.random.default_rng(40 + 2 * prec + inverse)
    npdt = np.complex128 if prec == F64 else np.complex64
    xh = (rng.standard_normal((nx, n, n)) + 1j * rng.standard_normal((nx, n, n))).astype(npdt)
    x = torch.from_numpy(xh).cuda()
    out = nan_(torch.empty_like(x))
    c.arena.poison()
    c.run(out, x, direction)
    assert c.plan.lastLaunchCount() == (2 if c.fused else 3)
    c.check(out, c.want(x, direction), "exec")
    xl = xh.astype(np.clongdouble)
    ref = np.fft.fft if not inverse else (lambda v, axis: np.fft.ifft(v, axis=axis) * v.shape[axis])
    for axis in ((2, 1, 0) if not inverse else (0, 1, 2)):
        xl = ref(xl, axis=axis)
    s = spec(prec, (nx, n, n))
    rel, mx = error_check(s, out.cpu().numpy(), xl)
    key = ("f64" if prec == F64 else "f32", "inverse" if inverse else "forward")
    print(f"long double {key} {nx}x{n}x{n}: rel-L2 {rel:.2f}, max {mx:.2f} (units of u sqrt(sum log2 L))")
    assert rel <= 3 and mx <= 30, (rel, mx)
    c.destroy()


# ---- GPU: the batched small-field stage ----------------------------------------------------------------------------------------
class BatchCase:
    def __init__(self, n, prec, batch, inplace=False):
        self.n, self.prec, self.batch, self.inplace = n, prec, batch, inplace
        mk = lambda b, ip: _slab(n, prec, b, ip)  # noqa: E731
        self.plan = mk(batch, inplace)
        self.one = mk(1, False)
        self.seed = 77 * n + batch + 5 * prec + (1000 if inplace else 0)
        self.shape = (batch, n, n, n)

    def new_input(self):
        self.seed += 1
        return rand(self.shape, self.prec, self.seed)

    def want(self, x, direction):
        import torch

        out = torch.empty_like(x)
        for f in range(self.batch):
            self.one.execC2C(out[f], x[f], direction)
        torch.cuda.synchronize()
        return out

    def check_stage(self, inverse):
        order = ["x lines", "y lines", "z lines"] if inverse else ["z lines", "y lines", "x lines"]
        assert labels(live_schedule(self.plan, inverse)) == ["batched pass: " + o for o in order]

    def check(self, got, want, what):
        import torch

        torch.cuda.synchronize()
        assert not has_nan(got), f"{what}: NaN in the output"
        for f in range(self.batch):
            assert torch.equal(bits(got[f]), bits(want[f])), f"{what}: field {f} of {self.batch}: max |diff| {float((got[f] - want[f]).abs().max())}"

    def destroy(self):
        self.plan.destroy()
        self.one.destroy()


def _slab(n, prec, batch, inplace):
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double" if prec == F64 else "float", transform="c2c")
    plan.initFFT(dfft.GlobalSize(n, n, n), None, True, batch=batch, inplace=inplace)
    return plan


BATCH_CASES = [(n, prec) for n in (32, 64) for prec in (F64, F32)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,prec", BATCH_CASES)
@pytest.mark.parametrize("inplace", [False, True])
def test_batched_exec_after_exec(n, prec, inplace):
    """every batch size around the look-ahead, new input every exec, `out` (where the intermediate lives) NaN before every
    out-of-place exec; each field bit-identical to the unbatched plan"""
    import torch

    ahead = default_ahead(n, prec, device_l2(), fields=True)
    for batch in BATCH_SIZES(ahead):
        c = BatchCase(n, prec, batch, inplace)
        outs = [torch.empty(c.shape, dtype=cdt(prec), device="cuda") for _ in range(2)]
        for direction in (dfft.FORWARD, dfft.INVERSE):
            c.check_stage(1 if direction == dfft.INVERSE else 0)
            for i in range(3):
                x = c.new_input()
                want = c.want(x, direction)
                if inplace:
                    got = x.clone()
                    c.plan.execC2C(got, got, direction)
                else:
                    got = nan_(outs[i % 2])
                    c.plan.execC2C(got, x, direction)
                assert c.plan.lastLaunchCount() == 1
                c.check(got, want, f"batch {batch} (look-ahead {ahead}), direction {direction}, exec {i}")
        c.destroy()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("n,prec", BATCH_CASES)
def test_batched_graph_replay_between_eager_execs(n, prec):
    """replays and eager execs alternating, each on a new input, `out` NaN before each, batch 2L + 1"""
    import torch

    ahead = default_ahead(n, prec, device_l2(), fields=True)
    c = BatchCase(n, prec, 2 * ahead + 1)
    s = torch.cuda.current_stream()
    cap_x = torch.empty(c.shape, dtype=cdt(prec), device="cuda")
    cap_out = torch.empty_like(cap_x)
    eager_out = [torch.empty_like(cap_x) for _ in range(2)]
    for direction in (dfft.FORWARD, dfft.INVERSE):
        x = c.new_input()
        c.plan.execC2C(nan_(eager_out[0]), x, direction, stream=s)
        c.check(eager_out[0], c.want(x, direction), "first eager exec")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            c.plan.execC2C(cap_out, cap_x, direction, stream=torch.cuda.current_stream())
        for i, kind in enumerate(["eager", "replay", "eager", "replay", "replay", "eager"]):
            x = c.new_input()
            want = c.want(x, direction)
            if kind == "replay":
                cap_x.copy_(x)
                nan_(cap_out)
                g.replay()
                got = cap_out
            else:
                got = nan_(eager_out[i % 2])
                c.plan.execC2C(got, x, direction, stream=s)
            c.check(got, want, f"direction {direction}, {kind} {i}")
        del g
    c.destroy()
    torch.cuda.empty_cache()


# ---- CPU: which shapes of the sweep run which stage ------------------------------------------------------------------------------
def dry_labels(shape, prec, inverse, batch=1, inplace=False):
    p = R.Plan(1, SL, shape, prec=prec, batch=batch if batch > 1 else None, inplace=inplace)
    return labels(R.describe(p, 0, inverse, 3))


def test_sweep_nx_at_50_mib():
    """the sweep's nx values for an H100's 50 MiB L2 (computed from the plan's rules, the table of the fused stage's
    smallest shapes and default look-aheads)"""
    want = {(512, F64): (13, 3), (512, F32): (26, 7), (256, F64): (51, 15), (256, F32): (101, 32)}
    for (n, prec), (smallest, ahead) in want.items():
        assert fused_nx("min", n, prec, DRY_L2) == smallest
        assert default_ahead(n, prec, DRY_L2) == ahead
    assert [default_ahead(n, prec, DRY_L2, fields=True) for n, prec in BATCH_CASES] == [32, 65, 3, 7]
    assert sorted({a for *_, a in SWEEP}) == sorted(AHEADS)


# (planes, precision) -> nx of the roles min, min+1, pow2, 100 at 50 MiB of L2, and the nx among them that do not fuse
SWEEP_AT_50_MIB = {(512, F64): ([13, 14, 64, 100], []), (512, F32): ([26, 27, 64, 100], []), (256, F64): ([51, 52, 64, 100], []),
                   (256, F32): ([101, 102, 128, 100], [100])}


@pytest.mark.parametrize("n,prec", PRECS)
def test_sweep_stages_at_50_mib(n, prec):
    """every (nx, planes, precision, batch, in place) the GPU tests run, with the step labels its plan lists: the fused
    stage everywhere except 100 planes of 256^2 f32 (exactly 50 MiB) and one plane below the smallest fused nx, with a
    Bluestein x pass wherever nx is not a power of two"""
    nxs, plain = SWEEP_AT_50_MIB[(n, prec)]
    assert [fused_nx(r, n, prec, DRY_L2) for r in ROLES] == nxs
    shapes = [(nx, 1, False) for nx in nxs] + [(fused_nx(r, n, prec, DRY_L2), b, ip) for n_, p_, r, b, ip in LAYOUTS if (n_, p_) == (n, prec)]
    for nx, batch, inplace in shapes:
        fused = nx not in plain
        assert fused == is_fused(nx, n, prec, DRY_L2)
        for inverse in (0, 1):
            p = R.Plan(1, SL, (nx, n, n), prec=prec, batch=batch if batch > 1 else None, inplace=inplace)
            steps = R.describe(p, 0, inverse, 3)["steps"]
            assert labels({"steps": steps}) == expected_labels(fused, inverse, batch), (nx, batch, inplace, inverse)
            assert all(s.get("n", 0) == (0 if nx & (nx - 1) == 0 else nx) for s in steps if s["label"] == "x pass")
    assert dry_labels((nxs[0] - 1, n, n), prec, 0) == PLAIN_FWD


@pytest.mark.parametrize("n,prec", BATCH_CASES)
def test_batched_sweep_runs_one_launch(n, prec):
    """every batch size the GPU tests run, in and out of place, lists the batched stage"""
    for batch in BATCH_SIZES(default_ahead(n, prec, DRY_L2, fields=True)):
        for inplace in (False, True):
            assert dry_labels((n, n, n), prec, 0, batch, inplace) == ["batched pass: z lines", "batched pass: y lines", "batched pass: x lines"]
            assert dry_labels((n, n, n), prec, 1, batch, inplace) == ["batched pass: x lines", "batched pass: y lines", "batched pass: z lines"]


@pytest.mark.parametrize("inverse", [0, 1])
def test_fused_bluestein_x_schedule_replay(inverse):
    """51 x 256 x 256 complex-double, the smallest fused shape with a non-power-of-two nx at 50 MiB of L2: the fused stage's
    two phases and the Bluestein x pass over the blocked hand-over, replayed on the CPU against the oracle"""
    assert dry_labels((51, 256, 256), F64, inverse) == expected_labels(True, inverse)
    assert run_case(1, SL, dfft.C2C, (51, 256, 256), 1, 1, P2P, SYNC, inverse, 3) < 1e-12
