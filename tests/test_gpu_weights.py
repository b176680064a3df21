"""Per-axis spectral weights on one GPU, f64 and f32: weighted execs against numpy (W * fftn(x), ifftn(W * X)) and against
the unweighted exec of the same plan times the broadcast W in torch; unit weights give the unweighted output; the x, y and
z derivatives of a trig polynomial from an R2C forward and a weighted C2R inverse; the input and a canary after the output
stay intact; re-pointed and rewritten weights on the next exec and on graph replay; multi-rank schedules replayed on one GPU
through dfft_debug_run_step."""
from __future__ import annotations

import math

import numpy as np
import pytest

import distributedfft_b200 as dfft
from oracle import dft_oracle as O

pytestmark = pytest.mark.gpu

CLASSES = {"slab": dfft.MPIcuFFT_Slab, "zyx": dfft.MPIcuFFT_Slab_Z_Then_YX, "pencil": dfft.MPIcuFFT_Pencil}
TOL = {True: 1e-12, False: 1e-5}  # rel-L2, f64 / f32

# name: (class, shape, transform, extra initFFT arguments)
CASES = {
    "slab_c2c": ("slab", (32, 64, 128), "c2c", {}),
    "slab_c2c_1024": ("slab", (1024, 16, 32), "c2c", {}),           # TILED x pass of 1024 points (register-fed when weighted)
    "slab_r2c": ("slab", (64, 32, 128), "r2c", {}),
    "zyx_r2c": ("zyx", (32, 64, 64), "r2c", {}),
    "pencil_c2c": ("pencil", (16, 32, 64), "c2c", {}),
    "bluestein": ("slab", (24, 20, 36), "c2c", {}),
    "padded_c2c": ("slab", (32, 32, 64), "c2c", {"spectral": (21, 20, 43)}),
    "padded_r2c": ("pencil", (32, 32, 64), "r2c", {"spectral": (21, 20, 42)}),
    "pruned_r2c": ("slab", (32, 32, 64), "r2c", {"data": (16, 17, 32)}),
    "batch_c2c": ("slab", (32, 32, 32), "c2c", {"batch": 2}),       # one-launch batched stage when unweighted
    "inplace_r2c": ("slab", (16, 32, 64), "r2c", {"inplace": True}),
}


def hermitian(w, half):
    """w made Hermitian along its axis: w[-k] = conj w[k] (half: the R2C z axis, real at 0 and at the Nyquist point)"""
    w = w.copy()
    if half:
        w[0], w[-1] = w[0].real, w[-1].real
        return w
    n = w.size
    neg = w[(-np.arange(n)) % n]
    return (w + np.conj(neg)) / 2


class Case:
    def __init__(self, name, f64):
        import torch

        kind, self.shape, self.transform, self.kw = CASES[name]
        self.c2c = self.transform == "c2c"
        self.f64 = f64
        self.batch = self.kw.get("batch", 1)
        self.plan = CLASSES[kind](dfft.Configurations(), dfft.Comm(), precision="double" if f64 else "float", transform=self.transform)
        self.plan.initFFT(dfft.GlobalSize(*self.shape), dfft.Partition(1, 1) if kind == "pencil" else None, True, **self.kw)
        self.rdt = torch.float64 if f64 else torch.float32
        self.cdt = torch.complex128 if f64 else torch.complex64
        self.spec = tuple(self.plan.getSpectralSize())
        self.data = tuple(self.kw.get("data", self.shape))
        self.klen = [self.spec[0], self.spec[1], self.spec[2] // 2 + 1 if not self.c2c else self.spec[2]]
        self.out_shape = tuple(self.plan.getOutSize())

    def weights(self, seed, herm=False):
        import torch

        rng = np.random.default_rng(seed)
        ws = []
        for a, n in enumerate(self.klen):
            w = rng.standard_normal(n) + 1j * rng.standard_normal(n)
            if herm and not self.c2c:
                w = hermitian(w, a == 2) if (a == 2 or self.spec[a] == self.shape[a]) else w
            ws.append(w)
        return ws, [torch.from_numpy(w).to(self.cdt).cuda() for w in ws]

    def run(self, out, x, inverse, stream=None):
        if self.c2c:
            self.plan.execC2C(out, x, dfft.INVERSE if inverse else dfft.FORWARD, stream=stream)
        elif inverse:
            self.plan.execC2R(out, x, stream=stream)
        else:
            self.plan.execR2C(out, x, stream=stream)

    def input(self, seed=3):
        rng = np.random.default_rng(seed)
        shp = (self.batch,) + self.data
        x = rng.standard_normal(shp) + (1j * rng.standard_normal(shp) if self.c2c else 0)
        return x

    def spectrum(self, x):
        """the unweighted numpy spectrum [field, K...] of the physical fields x"""
        out = []
        for f in range(self.batch):
            X = x[f]
            for axis in (2, 1, 0):
                half = not self.c2c and axis == 2
                pad = [(0, 0)] * 3
                pad[axis] = (0, self.shape[axis] - X.shape[axis])
                X = np.pad(X, pad)
                X = np.fft.rfft(X, axis=2) if half else np.fft.fft(X, axis=axis)
                pos = np.arange(self.spec[2] // 2 + 1) if half else np.fft.fftfreq(self.spec[axis], 1.0 / self.spec[axis]).astype(np.int64) % self.shape[axis]
                X = np.take(X, pos, axis=axis)
            out.append(X)
        return np.stack(out)

    def inverse_ref(self, X):
        out = []
        for f in range(self.batch):
            Y = X[f]
            for axis in (0, 1, 2):
                half = not self.c2c and axis == 2
                n = self.shape[axis]
                full = list(Y.shape)
                full[axis] = n // 2 + 1 if half else n
                E = np.zeros(full, dtype=np.result_type(Y.dtype, np.complex128))  # long double stays long double
                idx = [slice(None)] * 3
                idx[axis] = np.arange(self.spec[2] // 2 + 1) if half else np.fft.fftfreq(self.spec[axis], 1.0 / self.spec[axis]).astype(np.int64) % n
                E[tuple(idx)] = Y
                Y = np.fft.irfft(E, n=n, axis=2) * n if half else np.fft.ifft(E, axis=axis) * n
                Y = np.take(Y, np.arange(self.data[axis]), axis=axis)
            out.append(Y)
        return np.stack(out)

    def buffers(self, inverse, x):
        """(input tensor, output tensor with a canary field after the last) of a direction; the inverse input is the
        unweighted spectrum of x"""
        import torch

        if inverse:
            src = torch.from_numpy(self.spectrum(x)).to(self.cdt).cuda()
            if self.kw.get("inplace"):
                return src, None
            out = torch.full((self.batch + 1,) + self.data, 7.0, dtype=self.cdt if self.c2c else self.rdt, device="cuda")
        else:
            src = torch.from_numpy(x).to(self.cdt if self.c2c else self.rdt).cuda()
            if self.kw.get("inplace"):
                return src, None
            out = torch.full((self.batch + 1,) + tuple(self.klen), 7.0, dtype=self.cdt, device="cuda")
        return src, out

    def exec(self, inverse, src, out):
        """the output fields of one exec (in place: on a padded copy of src)"""
        import torch

        if self.kw.get("inplace"):
            nx, ny, nz = self.shape
            buf = torch.zeros((self.batch, nx, ny, nz // 2 + 1), dtype=self.cdt, device="cuda")
            real = torch.view_as_real(buf).view(self.batch, nx, ny, nz + 2)
            if inverse:
                buf.copy_(src)
                self.run(real, buf, 1)
                return real[..., :nz].clone()
            real[..., :nz] = src
            self.run(buf, real, 0)
            return buf.clone()
        self.run(out[:self.batch], src, inverse)
        return out[:self.batch].clone()


def broadcast(ws_t):
    return ws_t[0][:, None, None] * ws_t[1][None, :, None] * ws_t[2][None, None, :]


def rel(a, b):
    import torch

    return float(torch.linalg.vector_norm(a - b) / torch.linalg.vector_norm(b))


PARAMS = [(n, f64) for n in CASES for f64 in (True, False)]


@pytest.mark.parametrize("name,f64", PARAMS)
@pytest.mark.parametrize("inverse", [0, 1])
def test_weighted_exec(name, f64, inverse):
    """against numpy and against the unweighted exec times W; unit weights give the unweighted output; the input and
    the canary stay intact"""
    import torch

    ref = Case(name, f64)
    case = Case(name, f64)
    ws, ws_t = case.weights(11, herm=True)
    case.plan.setWeights(*ws_t)
    assert case.plan.getWeights()[0] is ws_t[0]
    x = case.input()
    src, out = case.buffers(inverse, x)
    keep = src.clone()
    got = case.exec(inverse, src, out)
    if out is not None:
        assert torch.equal(src, keep), "the input changed"
        assert (out[case.batch] == 7.0).all(), "the canary after the output changed"
    W = broadcast(ws_t)
    if inverse:
        plain = ref.exec(1, src * W, torch.empty_like(out) if out is not None else None)
        want_np = case.inverse_ref(case.spectrum(x) * np.multiply.outer(np.multiply.outer(ws[0], ws[1]), ws[2]))
    else:
        plain = ref.exec(0, src, torch.empty_like(out) if out is not None else None) * W
        want_np = case.spectrum(x) * np.multiply.outer(np.multiply.outer(ws[0], ws[1]), ws[2])
    assert rel(got, plain) < TOL[f64]
    # C2R of a truncated (padded) spectrum is not Hermitian, and numpy's irfft drops what the C2R pass does not: the
    # padded inverse is checked against the unweighted exec above only
    if not (inverse and not case.c2c and case.spec != case.shape):
        assert O.rel_l2(got.cpu().numpy(), want_np) < TOL[f64]
    # unit weights: exactly the unweighted output
    ones = [torch.ones(n, dtype=case.cdt, device="cuda") for n in case.klen]
    case.plan.setWeights(*ones)
    unit = case.exec(inverse, src, out)
    plain = ref.exec(inverse, src, torch.empty_like(out) if out is not None else None)
    assert torch.equal(unit, plain)
    case.plan.destroy()
    ref.plan.destroy()


@pytest.mark.parametrize("f64", [True, False])
def test_scale_and_null_axes(f64):
    """the output scale on top of the weights; an axis set to NULL is all ones; re-pointing takes effect on the next exec"""
    import torch

    case, ref = Case("pencil_c2c", f64), Case("pencil_c2c", f64)
    ws, ws_t = case.weights(4)
    case.plan.setWeights(ws_t[0], None, ws_t[2])
    case.plan.setScale(0.5, 0.25)
    x = case.input()
    src, out = case.buffers(0, x)
    got = case.exec(0, src, out)
    one = torch.ones_like(ws_t[1])
    want = ref.exec(0, src, torch.empty_like(out)) * broadcast([ws_t[0], one, ws_t[2]]) * 0.5
    assert rel(got, want) < TOL[f64]
    case.plan.setWeights(None, ws_t[1], None)
    got = case.exec(0, src, out)
    want = ref.exec(0, src, torch.empty_like(out)) * broadcast([torch.ones_like(ws_t[0]), ws_t[1], torch.ones_like(ws_t[2])]) * 0.5
    assert rel(got, want) < TOL[f64]
    case.plan.destroy()
    ref.plan.destroy()


def test_spectral_derivatives():
    """x, y and z derivatives of a trig polynomial: an R2C forward, then a C2R inverse weighted by i k (Nyquist zeroed)"""
    import torch

    nx, ny, nz = 32, 64, 128
    L = (2.0, 3.0, 5.0)
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="r2c")
    plan.initFFT(dfft.GlobalSize(nx, ny, nz), None, True)
    X, Y, Z = np.meshgrid(*(np.arange(n) * L[a] / n for a, n in enumerate((nx, ny, nz))), indexing="ij")
    kx, ky, kz = (2 * math.pi / L[a] for a in range(3))
    f = np.sin(3 * kx * X) * np.cos(2 * ky * Y) + np.cos(5 * kz * Z + 1.0) * np.sin(kx * X) + 0.5 * np.sin(7 * ky * Y + 4 * kz * Z)
    want = [3 * kx * np.cos(3 * kx * X) * np.cos(2 * ky * Y) + kx * np.cos(5 * kz * Z + 1.0) * np.cos(kx * X),
            -2 * ky * np.sin(3 * kx * X) * np.sin(2 * ky * Y) + 3.5 * ky * np.cos(7 * ky * Y + 4 * kz * Z),
            -5 * kz * np.sin(5 * kz * Z + 1.0) * np.sin(kx * X) + 2 * kz * np.cos(7 * ky * Y + 4 * kz * Z)]
    spec = torch.empty((nx, ny, nz // 2 + 1), dtype=torch.complex128, device="cuda")
    plan.execR2C(spec, torch.from_numpy(f).cuda())
    inv = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision="double", transform="r2c")
    inv.initFFT(dfft.GlobalSize(nx, ny, nz), None, True)
    ones = [torch.ones(n, dtype=torch.complex128, device="cuda") for n in (nx, ny, nz // 2 + 1)]
    w = [o.clone() for o in ones]
    inv.setWeights(*w)
    inv.setScale(1.0, 1.0 / (nx * ny * nz))
    out = torch.empty((nx, ny, nz), dtype=torch.float64, device="cuda")
    for a, n in enumerate((nx, ny, nz)):
        k = np.fft.fftfreq(n, 1.0 / n)[: (n // 2 + 1 if a == 2 else n)].copy()
        if a == 2:
            k = np.arange(n // 2 + 1, dtype=np.float64)
        k[n // 2] = 0.0  # the Nyquist entry of i k
        for b in range(3):  # rewrite the tables in place: the plan reads their contents at every exec
            w[b].copy_(torch.from_numpy(1j * (2 * math.pi / L[a]) * k).cuda() if b == a else ones[b])
        inv.execC2R(out, spec.clone())
        assert O.rel_l2(out.cpu().numpy(), want[a]) < 1e-12, a
    plan.destroy()
    inv.destroy()


@pytest.mark.parametrize("f64", [True, False])
def test_graph_replay(f64):
    """a graph keeps the pointers it was captured with and reads their contents at replay; setWeights needs an eager exec
    before the next capture"""
    import torch

    from distributedfft_b200._lib import DfftError

    case, ref = Case("slab_c2c", f64), Case("slab_c2c", f64)
    ws, ws_t = case.weights(8)
    case.plan.setWeights(*ws_t)
    x = case.input()
    src, out = case.buffers(0, x)
    case.exec(0, src, out)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            case.run(out[:1], src, 0, stream=s)
    plain = ref.exec(0, src, torch.empty_like(out))
    for k in range(2):
        for w in ws_t:
            w.mul_(1.5 if k else 1.0)
        g.replay()
        torch.cuda.synchronize()
        assert rel(out[:1], plain * broadcast(ws_t)) < TOL[f64]
    other = [w * 2 for w in ws_t]
    case.plan.setWeights(*other)
    g.replay()  # still the captured pointers
    torch.cuda.synchronize()
    assert rel(out[:1], plain * broadcast(ws_t)) < TOL[f64]
    with pytest.raises(DfftError):
        with torch.cuda.stream(s):
            g2 = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g2, stream=s):
                case.run(out[:1], src, 0, stream=s)
    got = case.exec(0, src, out)
    assert rel(got, plain * broadcast(other)) < TOL[f64]
    case.plan.destroy()
    ref.plan.destroy()


@pytest.mark.parametrize("P,decomp,shape,p1,p2,transform,extra", [
    (2, dfft.SLAB_ZY_THEN_X, (8, 16, 32), 2, 1, dfft.C2C, {}),
    (4, dfft.PENCIL, (8, 16, 32), 2, 2, dfft.R2C, {}),
    (4, dfft.SLAB_Z_THEN_YX, (12, 8, 20), 4, 1, dfft.C2C, {}),
    (8, dfft.PENCIL, (16, 16, 32), 2, 4, dfft.C2C, {"comm": 1, "batch": 2}),
    (8, dfft.SLAB_ZY_THEN_X, (16, 8, 64), 8, 1, dfft.R2C, {"spectral": (11, 8, 42)}),
])
@pytest.mark.parametrize("f64", [True, False])
@pytest.mark.parametrize("inverse", [0, 1])
def test_multi_rank_replay(P, decomp, shape, p1, p2, transform, extra, f64, inverse):
    import torch

    import step_replay as R
    import weights_replay as WR
    from test_weights import fwd_ref, inv_ref, random_weights

    p = R.Plan(P, decomp, shape, p1, p2, transform=transform, prec=dfft.F64 if f64 else dfft.F32, **extra)
    ws = random_weights(p, P + inverse)
    if transform == dfft.R2C:
        ws = tuple(hermitian(w, a == 2) for a, w in enumerate(ws))
    cdt = torch.complex128 if f64 else torch.complex64
    ws_t = [torch.from_numpy(w).to(cdt).cuda() for w in ws]
    rng = np.random.default_rng(7)
    real = transform == dfft.R2C
    xs = [rng.standard_normal(shape) + (0 if real else 1j * rng.standard_normal(shape)) for _ in range(p.fields)]
    if inverse:
        src = [fwd_ref(p, (None, None, None), x, 3) for x in xs]
        want = np.stack([inv_ref(p, ws, X, 3) for X in src])
    else:
        src, want = xs, np.stack([fwd_ref(p, ws, x, 3) for x in xs])
    dt = np.float64 if f64 else np.float32
    src = [s.astype(np.result_type(s.dtype, dt)) if np.iscomplexobj(s) else s.astype(dt) for s in src]
    if not f64:
        src = [s.astype(np.complex64) if np.iscomplexobj(s) else s for s in src]
    got = WR.gpu_output(p, ws_t, inverse, 3, src)
    assert O.rel_l2(got, want) < TOL[f64]
