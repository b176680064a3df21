"""Accuracy of every unit a caller treats as independent, against a long-double reference, at every kernel length.

A unit is a field of a batch, a component of an interleaved plan, or a line of the single-axis entry points.  Each unit is
held to the bounds of test_gpu_schedule_replay on its own norm: rel-L2 <= 3 and max |err| <= 30 rms(unit), both in units of
u sqrt(sum log2 L) (u the unit roundoff of the plan's precision, L the power-of-two length each transformed axis runs, M on
Bluestein axes).  The inputs mix magnitudes across units: unit i is scaled by 1, 2^20, 2^-20 or 0 in turn, so neighbouring
units differ by about 10^6, and a unit whose input is zero must come out as exact zeros.  The reference is numpy's FFT in
long double (scipy's DCT / DST for R2R) on the exact values that went to the device.  Every case also checks that the input
is unchanged, that a canary after the output is untouched, and that no output element is still the NaN the output buffer
starts as.

Families:
  1. interleaved plans (C components per point), per component: C2C with Nz = 2..8192 on (4, 2, Nz) and (2, 3, Nz) (a
     Bluestein y axis), R2C / C2R with Nz = 4..8192; C on both sides of every tile width, d = 1, 2, 3, both directions,
     f32 and f64, a scale != 1 per length;
  2. padded plans, per field (batch 3): every N = 2..8192 on z (R2C up to 16384), and on x with narrow and wide tiles,
     K in {1, 2, ceil(N/2), N/2 + 1, N - 1}; the x pass's column count B is above the narrow tile width of the length
     (asserted from dfft_plan_describe) and leaves a part-full tile;
  3. the single-axis entry points, per line: dfft_fft1d_contig (C2C, R2C, C2R) and dfft_fft1d_general (default, TMA-fed,
     narrow and wide tiles) at every length, Bluestein lengths 2^k +- 1, 3 and 5, with line and column counts that leave
     partial CTAs and tiles;
  4. the one-launch batched stage (32^3 and 64^3) and 3D DCT / DST / R2HC plans, per field;
  5. dfft_fft1d_r2r, per line, against the larger norm of the line pair its kernel transforms together (lines 2L, 2L + 1
     of CONTIG, columns 2c, 2c + 1 of TILED): the R2R kernels run two real lines as one complex line, so a line's error
     follows its partner's magnitude.  A zero pair gives exact zeros;
  6. (CPU) the paired split the interleaved R2C / C2R pass once used (components c, c + 1 as z = x_c + i x_{c+1}) fails
     the per-unit bound when the partner is 2^20 times larger, in both precisions; a line on its own passes.

Worst errors measured over this module on an H100 80GB HBM3 (700 W), in units of u sqrt(sum log2 L), rel-L2 / max over
rms(unit), f64 then f32:
  interleaved C2C 1.07 / 3.8, 0.92 / 4.3;  interleaved R2C / C2R 0.66 / 4.4, 0.67 / 4.5;
  padded z C2C 0.68 / 3.0, 0.66 / 3.3;  padded z R2C / C2R 0.73 / 3.9, 0.76 / 3.8;
  padded x C2C 0.76 / 3.3, 0.69 / 3.0;  padded x R2C / C2R 0.81 / 4.2, 0.70 / 4.1;
  1D contig C2C 1.62 / 4.3, 1.55 / 4.4;  R2C 1.08 / 3.0, 0.97 / 3.9;  C2R 1.10 / 3.5, 1.08 / 4.1;
  1D general, powers of two 0.96 / 3.1, 0.96 / 3.5;  Bluestein 1.42 / 4.8, 1.55 / 4.9;
  batched stage 0.65 / 3.3, 0.68 / 3.2;  3D R2R plans 0.70 / 5.1, 0.75 / 5.1;
  1D R2R against the pair's norm: CONTIG 1.71 / 4.9, 1.42 / 4.4;  TILED 1.85 / 5.5, 1.44 / 3.9.
The bounds (3 and 30) hold every family.  With the paired split the interleaved R2C / C2R pass used before, that family
missed the rel-L2 bound by a factor of 2.7e4 to 1.4e5 in both precisions.  The module takes about 85 s on the H100; the
long-double references of the interleaved family, the largest, take about 26 s of CPU time."""
import json
import math

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
from test_gpu_schedule_replay import UNIT, error_check, run_lengths, same_bits
from test_gpu_transform_axes import canary_ok, canary_out
from test_padded import fwd_ref as padded_fwd, inv_ref as padded_inv
from step_replay import describe_raw
from test_r2r_mixed import r2r_1d
from test_transform_axes import fwd_ref, inv_ref

F32, F64 = dfft.F32, dfft.F64
C2C, R2C, DCT, DST, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.DST, dfft.R2HC
NPR = {F64: np.float64, F32: np.float32}
NPC = {F64: np.complex128, F32: np.complex64}
TR = {F64: torch.float64, F32: torch.float32}
TC = {F64: torch.complex128, F32: torch.complex64}
PNAME = {F64: "double", F32: "float"}
PRECS = [F64, F32]
PIDS = ["f64", "f32"]
ALL = (1, 1, 1)
REL_BOUND, MAX_BOUND = 3.0, 30.0
SCALES = (1.0, 2.0 ** 20, 2.0 ** -20, 0.0)
# R2R lines pair up: (1, 2^20) and (2^-20, 0) mix magnitudes within a pair, (0, 0) is a zero pair
R2R_SCALES = (1.0, 2.0 ** 20, 2.0 ** -20, 0.0, 0.0, 0.0)
CAP = 1 << 20  # values per case
POW2 = [1 << k for k in range(1, 14)]
BLUESTEIN = [3, 5] + [n for k in range(3, 13) for n in ((1 << k) - 1, (1 << k) + 1) if n <= 4095]
WORST = {}  # (family, precision) -> worst (rel-L2, max)


def spec(prec, shape, d=3):
    """the fields error_check and run_lengths read"""
    return dict(prec=prec, shape=tuple(shape), d=d, axes=ALL)


def shape_of(prec, log2n):
    """Shape<T, LOG2N>'s tile constants (fft_kernels.cuh): (TBC lines per CONTIG CTA, TBT tile width, TBT_WIDE)"""
    esz = 16 if prec == F64 else 8
    log2e = min(log2n, 4)
    tpl = 1 << (log2n - log2e)
    ct = 128 if prec == F64 and log2n >= 9 else 256
    tbc = min(max(ct // tpl, 1), 64)
    minrow = 64 // esz
    want = 4096 >> log2n
    tbt_ = minrow if want < minrow else min(want, 32)
    cap = min((128 * 1024) // ((1 << log2n) * esz), 1024 // tpl)
    tbt = max(cap, 1) if tbt_ > cap else tbt_
    wide = 2 * tbt if 2 * tbt <= cap and 2 * tbt <= 32 else tbt
    return tbc, tbt, wide


def run_log2(n):
    """log2 of the power-of-two length an n-point C2C line runs (M for Bluestein lengths)"""
    return n.bit_length() - 1 if n & (n - 1) == 0 else (2 * n - 2).bit_length()


def unit_scales(count, off=0, cycle=SCALES):
    return np.array([cycle[(i + off) % len(cycle)] for i in range(count)])


def mixed(shape, axis, prec, complex_, seed, off=0, cycle=SCALES):
    """normal values in the plan's precision with unit i along `axis` scaled by cycle[i + off]; (values, unit scales)"""
    rng = np.random.default_rng(seed)
    v = rng.standard_normal(shape)
    if complex_:
        v = v + 1j * rng.standard_normal(shape)
    s = unit_scales(shape[axis], off, cycle)
    v = v * s.reshape([-1 if a == axis else 1 for a in range(len(shape))])  # powers of two: exact
    return v.astype((NPC if complex_ else NPR)[prec]), s


def ld(x):
    return x.astype(np.clongdouble if np.iscomplexobj(x) else np.longdouble)


def on_device(fn, x, out_shape, out_dtype):
    """fn(out, inp) on a device copy of x, into a NaN-filled output followed by a canary; the output as numpy"""
    inp = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    n = int(np.prod(out_shape))
    buf = canary_out(n, out_dtype)
    buf[:n] = float("nan")
    fn(buf[:n].view(tuple(out_shape)), inp)
    torch.cuda.synchronize()
    assert canary_ok(buf), "the element after the output was written"
    assert same_bits(inp.cpu().numpy(), np.ascontiguousarray(x)), "the input changed"
    got = buf[:n].view(tuple(out_shape)).cpu().numpy()
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements were never written"
    return got


def note(family, prec, rel, mx, worst=WORST):
    key = (family, "f64" if prec == F64 else "f32")
    w = worst.get(key, (0.0, 0.0))
    worst[key] = (max(w[0], rel), max(w[1], mx))


def check_units(family, s, got, ref, axis, scales, what="", worst=WORST):
    """the per-unit bounds, unit i being index i along `axis`; scales[i] == 0: the unit must be exact zeros.  The worst
    errors go to `worst` (the calling module's report)"""
    g, r = np.moveaxis(got, axis, 0), np.moveaxis(np.asarray(ref), axis, 0)
    for i in range(r.shape[0]):
        if scales[i] == 0:
            assert not np.any(g[i]), f"{family} {what}: unit {i} has a zero input but a nonzero output"
            continue
        rel, mx = error_check(s, g[i], r[i])
        note(family, s["prec"], rel, mx, worst)
        assert rel <= REL_BOUND and mx <= MAX_BOUND, \
            f"{family} {what}: unit {i} of {r.shape[0]} (input scale {scales[i]:g}): rel-L2 {rel:.2f}, max {mx:.2f} u sqrt(sum log2 L)"


def check_pairs(family, s, got, ref, axis, scales, what=""):
    """the per-line bounds relative to the larger norm of the pair (2i, 2i + 1) along `axis` (a lone last line: a zero
    partner); a zero pair must be exact zeros"""
    unit = UNIT[s["prec"]] * math.sqrt(max(1.0, sum(math.log2(n) for n in run_lengths(s))))
    g, r = np.moveaxis(got, axis, 0), np.moveaxis(np.asarray(ref), axis, 0)
    norms = [float(np.sqrt(np.sum(np.abs(r[i]) ** 2))) for i in range(r.shape[0])]
    for i in range(r.shape[0]):
        p = i ^ 1
        if scales[i] == 0 and (p >= len(scales) or scales[p] == 0):
            assert not np.any(g[i]), f"{family} {what}: line {i} and its partner are zero but the output is not"
            continue
        big = max(norms[i], norms[p] if p < len(norms) else 0.0)
        err = g[i].astype(r.dtype) - r[i]
        rel = float(np.sqrt(np.sum(np.abs(err) ** 2))) / big / unit
        mx = float(np.max(np.abs(err))) / (big / math.sqrt(r[i].size)) / unit
        note(family, s["prec"], rel, mx)
        assert rel <= REL_BOUND and mx <= MAX_BOUND, \
            f"{family} {what}: line {i} (scale {scales[i]:g}, partner's larger norm): rel-L2 {rel:.2f}, max {mx:.2f} u sqrt(sum log2 L)"


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if WORST:
        print("\nworst error per unit, in u sqrt(sum log2 L) (rel-L2 bound 3, max bound 30):")
        for (fam, prec), (rel, mx) in sorted(WORST.items()):
            print(f"  {fam:24s} {prec}: rel-L2 {rel:.3f}  max {mx:.3f}")


def plan_of(prec, transform, shape, **kw):
    plan = dfft.MPIcuFFT_Slab(dfft.Configurations(), dfft.Comm(), precision=PNAME[prec], transform=transform)
    plan.initFFT(dfft.GlobalSize(*shape), None, True, **kw)
    return plan


def exact_scale(prec, s):
    """the scale as the kernels apply it: rounded to the plan's precision once"""
    return np.longdouble(float(np.float32(s)) if prec == F32 else s)


# ---- 1. interleaved plans, per component ----------------------------------------------------------------------------------
ILV_C = (2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 64)


def interleaved_case(transform, grid, lg):
    nz = 1 << lg
    r2c = transform == "r2c"
    t = R2C if r2c else C2C
    family = "interleaved " + ("R2C/C2R" if r2c else "C2C")
    for ci, comps in enumerate(ILV_C):
        nx, ny = grid
        if nx * ny * nz * comps > CAP:
            if ny % 2:
                continue  # keep the Bluestein y axis, skip this C
            nx, ny = 2, 2  # C = 64 at Nz = 8192 stays, on the smallest grid
        shape = (nx, ny, nz)
        scale = 1.0 / 3.0 if ci == lg % len(ILV_C) else None
        for inverse in (0, 1):
            k = ci + lg + inverse
            prec, d = PRECS[k % 2], 1 + k % 3
            plan = plan_of(prec, transform, shape, components=comps)
            try:
                if scale is not None:
                    plan.setScale(scale, scale)
                seed = lg * 1000 + ci * 10 + inverse
                if not inverse:
                    x, sc = mixed(shape + (comps,), 3, prec, not r2c, seed, off=ci)
                    ref = fwd_ref(ld(x), t, None, ALL, d)
                    out_shape, out_dt = tuple(plan.getPartialSize(d)) + (comps,), TC[prec]
                    fn = (lambda o, i: plan.execR2C(o, i, d)) if r2c else (lambda o, i: plan.execC2C(o, i, dfft.FORWARD, d))
                else:
                    if r2c:  # the half spectrum of real components
                        xr, sc = mixed(shape + (comps,), 3, prec, False, seed, off=ci)
                        x = fwd_ref(ld(xr), R2C, None, ALL, d).astype(NPC[prec])
                        assert x.shape[:3] == tuple(plan.getPartialSize(d))
                    else:
                        x, sc = mixed(shape + (comps,), 3, prec, True, seed, off=ci)
                    ref = inv_ref(ld(x), t, None, ALL, d, nz)
                    out_shape, out_dt = tuple(plan.getInSize()) + (comps,), TR[prec] if r2c else TC[prec]
                    fn = (lambda o, i: plan.execC2R(o, i, d)) if r2c else (lambda o, i: plan.execC2C(o, i, dfft.INVERSE, d))
                if scale is not None:
                    ref = ref * exact_scale(prec, scale)
                got = on_device(fn, x, out_shape, out_dt)
                check_units(family, spec(prec, shape, d), got, ref, 3, sc, f"{shape} C={comps} {'inv' if inverse else 'fwd'} d={d} {PIDS[k % 2]}")
            finally:
                plan.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("grid", [(4, 2), (2, 3)], ids=["4x2", "2x3"])
@pytest.mark.parametrize("lg", range(1, 14))
def test_interleaved_c2c(grid, lg):
    interleaved_case("c2c", grid, lg)


@pytest.mark.gpu
@pytest.mark.parametrize("lg", range(2, 14))
def test_interleaved_r2c_c2r(lg):
    interleaved_case("r2c", (4, 2), lg)


# ---- 2. padded plans, per field -------------------------------------------------------------------------------------------
def spectral_sizes(n):
    return sorted(k for k in {1, 2, (n + 1) // 2, n // 2 + 1, n - 1} if 1 <= k <= n)


def x_extent(transform, n):
    """(ny, nz) of the x cases: the x pass's column count B = ny nz (C2C) or ny (nz/2 + 1) (R2C) is above the narrow tile
    width TBT of both precisions and leaves the last tile part-full (C2C: a Bluestein y axis of 3, R2C: B = TBT + 2)"""
    tbt = max(shape_of(prec, n.bit_length() - 1)[1] for prec in PRECS)
    if transform == "r2c":
        return 2, max(tbt, 4)
    return 3, max(tbt // 2, 2)


def x_columns(transform, shape):
    return shape[1] * (shape[2] // 2 + 1 if transform == "r2c" else shape[2])


def padded_case(transform, axis, n):
    """batch 3 on a grid whose `axis` is n points long, for every K of spectral_sizes(n) on that axis"""
    r2c = transform == "r2c"
    t = R2C if r2c else C2C
    shape = (4, 2, n) if axis == 2 else (n,) + x_extent(transform, n)
    family = f"padded {'xyz'[axis]} " + ("R2C/C2R" if r2c else "C2C")
    for ki, kk in enumerate(spectral_sizes(n)):
        sp = list(shape)
        sp[axis] = kk
        for inverse in (0, 1):
            prec = PRECS[(ki + inverse) % 2]
            plan = plan_of(prec, transform, shape, batch=3, spectral=sp)
            try:
                if axis == 0:  # the x pass runs the intended columns, more than a narrow tile holds
                    _, tbt, wtile = shape_of(prec, n.bit_length() - 1)
                    xs = [st for st in json.loads(describe_raw(plan._h, inverse, 3))["steps"] if st["type"] == 0 and st["label"] == "x pass"]
                    assert xs and all(st["B"] == x_columns(transform, shape) > tbt for st in xs), (shape, [st["B"] for st in xs], tbt)
                seed = n * 100 + ki * 2 + inverse
                if not inverse:
                    x, sc = mixed((3,) + shape, 0, prec, not r2c, seed, off=ki)
                    ref = np.stack([padded_fwd(ld(x[f]), t, sp, 3) for f in range(3)])
                    out_shape, out_dt = (3,) + tuple(plan.getPartialSize(3)), TC[prec]
                    fn = (lambda o, i: plan.execR2C(o, i)) if r2c else (lambda o, i: plan.execC2C(o, i, dfft.FORWARD))
                else:
                    if r2c:  # the kept modes of real fields
                        xr, sc = mixed((3,) + shape, 0, prec, False, seed, off=ki)
                        x = np.stack([padded_fwd(ld(xr[f]), R2C, sp, 3) for f in range(3)]).astype(NPC[prec])
                        # an even K < N on x or y keeps -K/2 without +K/2: that mode alone is not the spectrum of a real
                        # field, and C2R defines no result for such input (numpy drops the imaginary parts, cuFFT
                        # leaves it undefined), so it is zeroed
                        for a in (0, 1):
                            if sp[a] < shape[a] and sp[a] % 2 == 0:
                                idx = [slice(None)] * 4
                                idx[a + 1] = sp[a] // 2
                                x[tuple(idx)] = 0
                    else:
                        x, sc = mixed((3,) + tuple(plan.getPartialSize(3)), 0, prec, True, seed, off=ki)
                    ref = np.stack([padded_inv(ld(x[f]), t, shape, sp, 3) for f in range(3)])
                    if r2c:
                        ref = ref.real
                    out_shape, out_dt = (3,) + tuple(plan.getInSize()), TR[prec] if r2c else TC[prec]
                    fn = (lambda o, i: plan.execC2R(o, i)) if r2c else (lambda o, i: plan.execC2C(o, i, dfft.INVERSE))
                got = on_device(fn, x, out_shape, out_dt)
                check_units(family, spec(prec, shape), got, ref, 0, sc, f"{shape} K={sp} {'inv' if inverse else 'fwd'} {PIDS[(ki + inverse) % 2]}")
            finally:
                plan.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("transform,lg", [("c2c", lg) for lg in range(1, 14)] + [("r2c", lg) for lg in range(2, 15)])
def test_padded_z(transform, lg):
    padded_case(transform, 2, 1 << lg)


@pytest.mark.gpu
@pytest.mark.parametrize("wide", ["1", "-1"])
@pytest.mark.parametrize("transform", ["c2c", "r2c"])
@pytest.mark.parametrize("lg", range(1, 14))
def test_padded_x(wide, transform, lg, monkeypatch):
    monkeypatch.setenv("DFFT_WIDE_TILES", wide)
    padded_case(transform, 0, 1 << lg)


# ---- 3. single-axis entry points, per line --------------------------------------------------------------------------------
def counts(tile):
    """1, and one fewer and one more than a CTA or tile holds"""
    return sorted({1, max(tile - 1, 1), tile + 1})


@pytest.mark.gpu
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_contig_c2c(prec):
    for n in POW2 + BLUESTEIN:
        tbc = shape_of(prec, run_log2(n))[0]
        s = spec(prec, (1, 1, n), 1)
        for lines in counts(tbc):
            for inverse in (0, 1):
                x, sc = mixed((lines, n), 0, prec, True, n * 7 + lines, off=inverse)
                ref = np.fft.ifft(ld(x), axis=1) * n if inverse else np.fft.fft(ld(x), axis=1)
                direction = dfft.INVERSE if inverse else dfft.FORWARD
                got = on_device(lambda o, i: dfft.fft1d_contig(prec, 0, direction, n, lines, o, n, i, n), x, (lines, n), TC[prec])
                check_units("1D contig C2C", s, got, ref, 0, sc, f"n={n} lines={lines} {'inv' if inverse else 'fwd'}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [1, 2], ids=["r2c", "c2r"])
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_contig_r2c_c2r(prec, kind):
    for lg in range(2, 15):
        n = 1 << lg
        h = n // 2 + 1
        s = spec(prec, (1, 1, n), 1)
        for lines in counts(shape_of(prec, lg - 1)[0]):
            xr, sc = mixed((lines, n), 0, prec, False, n * 3 + lines, off=kind)
            if kind == 1:
                ref = np.fft.rfft(ld(xr), axis=1)
                got = on_device(lambda o, i: dfft.fft1d_contig(prec, 1, dfft.FORWARD, n, lines, o, h, i, n), xr, (lines, h), TC[prec])
            else:
                x = np.fft.rfft(ld(xr), axis=1).astype(NPC[prec])
                ref = np.fft.irfft(ld(x), n=n, axis=1) * n
                got = on_device(lambda o, i: dfft.fft1d_contig(prec, 2, dfft.INVERSE, n, lines, o, n, i, h), x, (lines, n), TR[prec])
            check_units("1D contig " + ("R2C" if kind == 1 else "C2R"), s, got, ref, 0, sc, f"n={n} lines={lines}")


GENERAL_ENVS = [{}, {"DFFT_TMA": "1"}, {"DFFT_WIDE_TILES": "1"}, {"DFFT_WIDE_TILES": "-1"}]


@pytest.mark.gpu
@pytest.mark.parametrize("env", GENERAL_ENVS, ids=["default", "tma", "wide", "narrow"])
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_general(prec, env, monkeypatch):
    """[a0][n][b] arrays, b contiguous: units are the a0 x b lines along n, neighbouring columns of mixed magnitude"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    a0 = 2
    for n in POW2 + BLUESTEIN:
        _, tbt, wide = shape_of(prec, run_log2(n))
        s = spec(prec, (1, 1, n), 1)
        for b in sorted(set(counts(tbt)) | set(counts(wide))):
            for inverse in (0, 1):
                x, sc = mixed((a0 * b, n), 0, prec, True, n * 11 + b, off=inverse)
                x = np.ascontiguousarray(x.reshape(a0, b, n).transpose(0, 2, 1))  # unit (i, c) -> line i * b + c
                ref = np.fft.ifft(ld(x), axis=1) * n if inverse else np.fft.fft(ld(x), axis=1)
                direction = dfft.INVERSE if inverse else dfft.FORWARD
                st = (n * b, 0, b)
                got = on_device(lambda o, i: dfft.fft1d_general(prec, direction, n, a0, 1, b, o, st, i, st), x, (a0, n, b), TC[prec])
                flat = lambda a: a.transpose(0, 2, 1).reshape(a0 * b, n)  # noqa: E731
                family = "1D general " + ("Bluestein" if n & (n - 1) else "pow2")
                check_units(family, s, flat(got), flat(ref), 0, sc, f"n={n} b={b} {'inv' if inverse else 'fwd'} {env}")


# ---- 4. other stages, per field -------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("n", [32, 64])
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_batched_stage(prec, n):
    """the one-launch stage of batched small cubes"""
    shape, batch = (n, n, n), 4
    plan = plan_of(prec, "c2c", shape, batch=batch)
    try:
        for inverse in (0, 1):
            x, sc = mixed((batch,) + shape, 0, prec, True, n + inverse, off=inverse)
            ref = np.stack([np.fft.ifftn(ld(x[f])) * n ** 3 if inverse else np.fft.fftn(ld(x[f])) for f in range(batch)])
            direction = dfft.INVERSE if inverse else dfft.FORWARD
            got = on_device(lambda o, i: plan.execC2C(o, i, direction), x, x.shape, TC[prec])
            assert plan.lastLaunchCount() == 1, "not the one-launch stage"
            check_units("batched stage", spec(prec, shape), got, ref, 0, sc, f"{n}^3 {'inv' if inverse else 'fwd'}")
    finally:
        plan.destroy()


R2R_PLANS = {"dct": (DCT,) * 3, "dst": (DST,) * 3, "r2hc": (R2HC,) * 3}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(R2R_PLANS))
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_r2r_plans(prec, name):
    """3D DCT / DST / R2HC plans, batch 3: each field on its own norm (line pairs stay within a field)"""
    kinds = R2R_PLANS[name]
    shape = (8, 16, 32)
    plan = plan_of(prec, name if name != "r2hc" else ("r2hc",) * 3, shape, batch=3)
    try:
        for d in (1, 3):
            for inverse in (0, 1):
                x, sc = mixed((3,) + shape, 0, prec, False, d * 10 + inverse, off=d + inverse)
                ref = np.stack([(inv_ref(ld(x[f]), None, kinds, ALL, d, shape[2]) if inverse else fwd_ref(ld(x[f]), None, kinds, ALL, d))
                                for f in range(3)])
                direction = dfft.INVERSE if inverse else dfft.FORWARD
                got = on_device(lambda o, i: plan.execR2R(o, i, direction, d), x, x.shape, TR[prec])
                check_units("3D R2R plan", spec(prec, shape, d), got, ref, 0, sc, f"{name} d={d} {'inv' if inverse else 'fwd'}")
    finally:
        plan.destroy()


# ---- 5. R2R line pairing, pinned ------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("kind", [DCT, DST, R2HC], ids=["dct", "dst", "r2hc"])
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_r2r_lines(prec, kind):
    for lg in range(1, 14):
        n = 1 << lg
        tbc, tbt, _ = shape_of(prec, lg)
        s = spec(prec, (1, 1, n), 1)
        for inverse in (0, 1):
            direction = dfft.INVERSE if inverse else dfft.FORWARD
            # CONTIG: a lines (b = 1), TBC line pairs per CTA
            for a in sorted({6, 2 * tbc + 1}):
                x, sc = mixed((a, n), 0, prec, False, n + a + inverse, cycle=R2R_SCALES)
                ref = r2r_1d(ld(x), kind, bool(inverse), 1)
                got = on_device(lambda o, i: dfft.fft1d_r2r(prec, kind, direction, n, a, 1, o, i), x, (a, n), TR[prec])
                check_pairs("1D R2R contig (pair)", s, got, ref, 0, sc, f"n={n} lines={a} {'inv' if inverse else 'fwd'}")
            # TILED: [2][n][b], TBT column pairs per tile
            for b in sorted({6, 2 * tbt + 1}):
                x, sc = mixed((2, b, n), 1, prec, False, n + b + inverse + 7, cycle=R2R_SCALES)
                x = np.ascontiguousarray(x.transpose(0, 2, 1))
                ref = r2r_1d(ld(x), kind, bool(inverse), 1)
                got = on_device(lambda o, i: dfft.fft1d_r2r(prec, kind, direction, n, 2, b, o, i), x, (2, n, b), TR[prec])
                for row in range(2):
                    check_pairs("1D R2R tiled (pair)", s, got[row], ref[row], 1, sc, f"n={n} b={b} row={row} {'inv' if inverse else 'fwd'}")


# ---- 6. the paired split, emulated on the CPU -----------------------------------------------------------------------------
def split_emulation(a, b, prec):
    """X_a of the real lines a when they ride one complex FFT of the plan's precision as z = a + i b (b = None: alone),
    split as (Z[k] + conj Z[-k]) / 2 — the arithmetic of the interleaved R2C pass before each component got its own line"""
    z = (a + 1j * (b if b is not None else 0)).astype(NPC[prec])
    Z = np.fft.fft(z, axis=-1)  # numpy >= 2 keeps complex64 in complex64
    Zm = np.conj(np.roll(Z[..., ::-1], 1, axis=-1))  # Z[-k mod N]
    n = a.shape[-1]
    return ((Z + Zm) * 0.5)[..., :n // 2 + 1]


def worst_line(s, got, ref):
    errs = [error_check(s, got[i], ref[i]) for i in range(ref.shape[0])]
    return max(e[0] for e in errs), max(e[1] for e in errs)


@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_paired_split_fails_the_per_unit_bound(prec):
    """64 lines of 256 points whose partner lines are 2^20 times larger: the paired split's error follows the partner's
    norm (u |x_b|, not u |x_a|) and fails the bound; the same line transformed on its own passes it"""
    rng = np.random.default_rng(3)
    a = rng.standard_normal((64, 256)).astype(NPR[prec])
    b = (rng.standard_normal((64, 256)) * 2.0 ** 20).astype(NPR[prec])
    s = spec(prec, (1, 1, 256), 1)
    ref = np.fft.rfft(ld(a), axis=1)
    paired = split_emulation(a, b, prec)
    assert paired.dtype == NPC[prec]
    rel, mx = worst_line(s, paired, ref)
    assert rel > 100 * REL_BOUND and mx > MAX_BOUND, (rel, mx)
    rel, mx = worst_line(s, split_emulation(a, None, prec), ref)
    assert rel <= REL_BOUND and mx <= MAX_BOUND, (rel, mx)
