"""Accuracy of the weighted and pruned pass kernels against a long-double reference, per field, at every kernel length and
tile width.

The units, bounds and inputs are those of test_gpu_accuracy's family 2: batch 3, field i scaled by 1, 2^20, 2^-20 or 0 in
turn, each field held to rel-L2 <= 3 and max |err| <= 30 rms(field) in units of u sqrt(sum log2 L), and a zero field must
come out as exact zeros.  The reference is numpy in long double (test_weights.fwd_ref / inv_ref) on the exact inputs and
on the weight tables as the device holds them (rounded to the plan's precision).  C2R inputs are spectra of real fields
with the unpaired -K/2 mode of an even K < N zeroed, and their weights are Hermitian per axis (real at z = 0 and at the
Nyquist point).

Families:
  W1. weighted z passes: (4, 2, N), C2C N = 2..8192, R2C / C2R N = 4..16384 (M = 2..8192: both C2R builds), all three
      axes weighted; the plain plan, a padded plan per K in {1, 2, ceil(N/2), N/2 + 1, N - 1}, a pruned plan per M in
      {1, 2, N/2, N/2 + 1, N - 1} (rounded down to even on an R2C z axis), and one plan with a data hole and a spectral
      hole on z at once; partial d and a kept x axis at some lengths;
  W2. weighted x passes: N on x (C2C and R2C plans) with DFFT_WIDE_TILES = 1 and -1, the same K / M sets, y and z
      extents chosen so the x pass's column count B is next to the narrow and the wide tile width (partial tiles; B
      > TBT for wide runs, asserted from dfft_plan_describe);
  W3. weighted Bluestein passes: C2C, n = 3, 5, 2^k +- 1 <= 4095 on z (CONTIG) and on x (TILED, a partial tile);
  P1. pruned plans without weights (the padded twins with a physical hole): the z and x sweeps of W1 / W2 with the same
      M sets, with and without a K on the same axis; the z sweep prunes x to 3 of 4 points and runs d = 1, 2, 3, so an
      untransformed pruned axis keeps its M points.
Beside the bounds, every case checks exactly:
  - weights: every table of 8 or more entries is zero at the edges of its view (0, ceil(L/2) - 1, ceil(L/2), L - 1 and,
    for C2R, their Hermitian partners), and a forward output at such an index is exactly zero in every field;
  - each table sits in a larger CUDA buffer between NaN guards, and the tables of axes an exec does not transform
    (partial d, kept axes) are all NaN, so a read outside a table or of a table that must not be read shows as NaN;
  - all-ones weights give the same values (+-0 alike) as the unweighted plan of the same shape, K and M;
  - the scale rule: an exec with scale 1/3 is the scale-1 exec times 1/3 element by element, rounded in the plan's
    precision.
A CPU test derives every (precision, log2 n, kind) the weighted cases launch from dfft_plan_describe and the tile rule
of launch_twin, and asserts that every weighted twin is among them: CONTIG, narrow and wide TILED (where the widths
differ), R2C, the C2R warp-shuffle (M <= 512) and shared-memory builds, and Bluestein CONTIG / TILED for each M.  Other
CPU tests emulate plausible index defects with numpy and show that the per-field bound rejects them, and check the
reference against dense DFT matrices.

Worst errors measured over this module on an H100 80GB HBM3 (700 W), in units of u sqrt(sum log2 L), rel-L2 / max over
rms(field), f64 then f32:
  W1 weighted z C2C 0.94 / 11.5, 0.95 / 10.1;  W1 weighted z R2C / C2R 1.24 / 9.4, 2.19 / 9.0;
  W2 weighted x C2C 1.04 / 12.3, 1.09 / 10.8;  W2 weighted x R2C / C2R 1.65 / 11.3, 1.12 / 10.4;
  W3 weighted Bluestein z 1.05 / 13.2, 1.04 / 11.1;  W3 weighted Bluestein x 1.05 / 13.4, 1.17 / 10.2;
  P1 pruned z C2C 0.89 / 3.4, 0.72 / 3.1;  P1 pruned z R2C / C2R 0.81 / 4.0, 0.86 / 4.6;
  P1 pruned x C2C 0.82 / 3.1, 0.89 / 3.3;  P1 pruned x R2C / C2R 0.63 / 3.7, 0.65 / 3.7.
The weighted families' max errors are about three times those of the unweighted ones, well within the bound.  The bounds (3 and 30) hold every family, every exact check holds at every case, and all-ones weights matched the
unweighted plans everywhere.  With the C2R shared-memory build's partner weight taken as w[k] instead of w[M - k], W1
fails at every R2C / C2R length that runs that build (N = 2048..16384) by a factor of 10^6 (f32) to 10^15 (f64) in
rel-L2, and passes at the shorter ones.  The module takes about 75 s on the H100."""
from __future__ import annotations

import json
import math
from typing import NamedTuple

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
import step_replay as R
import weights_replay as WR
from test_gpu_accuracy import (BLUESTEIN, CAP, MAX_BOUND, NPC, NPR, PIDS, PRECS, REL_BOUND, TC, TR, check_units, counts, exact_scale,
                               ld, mixed, on_device, plan_of, run_log2, shape_of, spec, spectral_sizes)
from test_gpu_schedule_replay import error_check
from test_gpu_weights import hermitian
from test_weights import fwd_ref, inv_ref, transformed

F32, F64 = dfft.F32, dfft.F64
WORST = {}  # (family, precision) -> worst (rel-L2, max)
SCALE = 1.0 / 3.0
GUARD = 4  # NaN elements before and after each table
MIN_ZEROS = 8  # tables shorter than this keep every entry nonzero (their edges would be most of the table)


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if WORST:
        print("\nworst error per field, in u sqrt(sum log2 L) (rel-L2 bound 3, max bound 30):")
        for (fam, prec), (rel, mx) in sorted(WORST.items()):
            print(f"  {fam:24s} {prec}: rel-L2 {rel:.3f}  max {mx:.3f}")


# ---- cases ----------------------------------------------------------------------------------------------------------------
class Case(NamedTuple):
    family: str
    transform: str  # "c2c" / "r2c"
    shape: tuple
    spectral: tuple | None
    data: tuple | None
    d: int
    axes: tuple | None  # transform axes (x, y, z); None: all
    inverse: int
    prec: int
    weighted: bool
    env: str | None  # DFFT_WIDE_TILES
    scaled: bool  # the scale-1/3 exec is held to the bounds too (the scale rule is checked on every case)
    seed: int
    B: int | None = None  # the x pass's column count the grid was chosen for

    def plan(self):
        """the geometry of the case as step_replay describes it (the references read its shape, spectral, data, axes)"""
        return R.Plan(1, dfft.SLAB_ZY_THEN_X, self.shape, transform=dfft.R2C if self.transform == "r2c" else dfft.C2C, prec=self.prec,
                      batch=3, spectral=self.spectral, data=self.data, axes=self.axes)

    def what(self):
        return (f"{self.transform} {self.shape} K={self.spectral} M={self.data} d={self.d} axes={self.axes} "
                f"{'inv' if self.inverse else 'fwd'} {PIDS[PRECS.index(self.prec)]} wide={self.env}")


def data_sizes(n, pairs=False):
    """the pruned extents of an n-point axis: {1, 2, n/2, n/2 + 1, n - 1}, rounded down to even on an R2C z axis (pairs)"""
    ms = {1, 2, n // 2, n // 2 + 1, n - 1}
    if pairs:
        ms = {m - m % 2 for m in ms}
    return sorted(m for m in ms if 1 <= m < n)


def hole_configs(n, pairs):
    """(K, M) of one axis: the plain plan, every K, every M, and one plan with both holes"""
    ks = [k for k in spectral_sizes(n) if k < n]
    ms = data_sizes(n, pairs)
    out = [(None, None)] + [(k, None) for k in ks] + [(None, m) for m in ms]
    if ks and ms:
        out.append((ks[len(ks) // 2], ms[-1]))
    return out


def with_axis(shape, axis, v):
    if v is None:
        return None
    s = list(shape)
    s[axis] = v
    return tuple(s)


# x-pass grids: (ny, nz) by the x pass's column count B = ny nz (C2C) or ny (nz / 2 + 1) (R2C).  C2C axes are powers of two
# >= 2 or any length >= 3 (Bluestein); R2C axes are powers of two, z >= 4.
def _grids(transform):
    g = {}
    if transform == "r2c":
        for nz in (4, 8, 16, 32, 64):
            for ny in (2, 4, 8, 16, 32):
                g.setdefault(ny * (nz // 2 + 1), (ny, nz))
    else:
        for b in range(4, 65):
            if b % 2 == 0:
                g[b] = (2, b // 2)
            elif b % 3 == 0 and b >= 9:
                g[b] = (3, b // 3)
    return dict(sorted(g.items()))


GRIDS = {t: _grids(t) for t in ("c2c", "r2c")}


def realize(transform, t, tbt):
    """the reachable B nearest to t on t's side of the tile width tbt: <= t when t <= tbt, >= t otherwise"""
    bs = list(GRIDS[transform])
    below, above = [b for b in bs if b <= t], [b for b in bs if b >= t]
    if t <= tbt and below:
        return below[-1]
    return above[0] if above else bs[-1]


def x_widths(transform, prec, n):
    """the column counts of the x cases: next to the narrow and the wide tile width, within CAP values per case"""
    _, tbt, wide = shape_of(prec, n.bit_length() - 1)
    bs = {realize(transform, t, tbt if t <= tbt else wide) for t in set(counts(tbt)) | set(counts(wide))}
    return sorted(b for b in bs if 3 * n * b <= CAP) or [min(GRIDS[transform])]


def wide_widths(transform, prec, n):
    """the column counts of wide runs: those of x_widths above the narrow tile width where the widths differ"""
    _, tbt, wide = shape_of(prec, n.bit_length() - 1)
    bs = x_widths(transform, prec, n)
    return bs if wide == tbt else [b for b in bs if b > tbt]


def x_grid(transform, n, b):
    ny, nz = GRIDS[transform][b]
    return (n, ny, nz)


def w1_cases(transform, lg):
    n = 1 << lg
    r2c = transform == "r2c"
    family = "W1 weighted z " + ("R2C/C2R" if r2c else "C2C")
    shape = (4, 2, n)
    cfgs = hole_configs(n, r2c)
    out = []
    for ci, (k, m) in enumerate(cfgs):
        for inverse in (0, 1):
            d = (3, 2, 1)[(lg + inverse) % 3] if ci == 0 else 3
            out.append(Case(family, transform, shape, with_axis(shape, 2, k), with_axis(shape, 2, m), d, None, inverse, PRECS[(ci + inverse + lg) % 2],
                            True, None, ci == lg % len(cfgs), lg * 1000 + ci * 10 + inverse))
    if lg % 3 == 0:  # a kept x axis: its table must not be read
        for inverse in (0, 1):
            out.append(Case(family, transform, shape, None, None, 3, (False, True, True), inverse, PRECS[(lg + inverse) % 2], True, None, False,
                            lg * 1000 + 999 - inverse))
    return out


def w2_cases(transform, lg, env):
    n = 1 << lg
    r2c = transform == "r2c"
    family = "W2 weighted x " + ("R2C/C2R" if r2c else "C2C")
    ei = ("1", "-1").index(env)
    out = []
    for ci, (k, m) in enumerate(hole_configs(n, False)):
        inverse, prec = (ci + ei) % 2, PRECS[(ci // 2 + lg) % 2]
        widths = wide_widths(transform, prec, n) if env == "1" else x_widths(transform, prec, n)
        b = widths[(ci + ei) % len(widths)]
        shape = x_grid(transform, n, b)
        out.append(Case(family, transform, shape, with_axis(shape, 0, k), with_axis(shape, 0, m), 3, None, inverse, prec, True, env, ci == 1,
                        lg * 1000 + ci * 10 + ei, b))
    return out


def w3_cases(axis):
    out = []
    for i, n in enumerate(BLUESTEIN):
        for inverse in (0, 1):
            prec = PRECS[(i + inverse) % 2]
            if axis == 2:
                shape, b = (4, 2, n), None
            else:
                _, tbt, _ = shape_of(prec, run_log2(n))
                b = realize("c2c", tbt + 1, tbt)
                shape = x_grid("c2c", n, b)
            out.append(Case(f"W3 weighted Bluestein {'xyz'[axis]}", "c2c", shape, None, None, 3, None, inverse, prec, True, None, i % 4 == 0,
                            n * 10 + inverse, b))
    return out


def p1_cases(transform, lg, axis):
    n = 1 << lg
    r2c = transform == "r2c"
    family = f"P1 pruned {'xyz'[axis]} " + ("R2C/C2R" if r2c else "C2C")
    ks = [k for k in spectral_sizes(n) if k < n] or [None]
    out = []
    for mi, m in enumerate(data_sizes(n, r2c and axis == 2)):
        for ki, k in enumerate((None, ks[mi % len(ks)])):
            ci = 2 * mi + ki
            if axis == 2:  # x pruned too: kept whole (3 points) where d < 3 leaves it untransformed
                shape, b, env = (4, 2, n), None, None
                inverses = (0, 1)
            else:
                env = ("1", "-1")[ci % 2]
                inverses = ((ci // 2) % 2,)
                widths = (wide_widths if env == "1" else x_widths)(transform, PRECS[(ci + inverses[0] + lg) % 2], n)
                b = widths[ci % len(widths)]
                shape = x_grid(transform, n, b)
            for inverse in inverses:
                data = with_axis(shape, axis, m)
                if axis == 2:
                    data = (3,) + data[1:]
                # d = 1, 2 on the z sweep only: an x case's x axis is transformed
                d = (3, 1, 2)[(ci + inverse + lg) % 3] if axis == 2 else 3
                out.append(Case(family, transform, shape, with_axis(shape, axis, k), data, d, None, inverse, PRECS[(ci + inverse + lg) % 2], False,
                                env, ci == 0, lg * 1000 + ci * 10 + inverse, b))
    return out


Z_LENGTHS = [("c2c", lg) for lg in range(1, 14)] + [("r2c", lg) for lg in range(2, 15)]
X_LENGTHS = [("c2c", lg) for lg in range(1, 14)] + [("r2c", lg) for lg in range(1, 14)]


def weighted_cases():
    out = [c for t, lg in Z_LENGTHS for c in w1_cases(t, lg)]
    out += [c for t, lg in X_LENGTHS for env in ("1", "-1") for c in w2_cases(t, lg, env)]
    return out + w3_cases(2) + w3_cases(0)


# ---- weights, inputs and references ---------------------------------------------------------------------------------------
def table_lengths(c):
    k = c.spectral or c.shape
    return [k[0], k[1], k[2] // 2 + 1 if c.transform == "r2c" else k[2]]


def read_axes(c):
    """the axes whose tables the exec reads: the transformed ones among its first d"""
    return transformed(c.plan(), c.d)


def zero_indices(length, herm):
    """the edges of a table's view, and their Hermitian partners where the table must stay Hermitian"""
    if length < MIN_ZEROS:
        return []
    e = {0, (length + 1) // 2 - 1, (length + 1) // 2, length - 1}
    if herm:
        e |= {(length - m) % length for m in e}
    return sorted(e)


def tables(c):
    """per axis: the table as the device holds it (numpy, the plan's precision; all NaN where it must not be read) and its
    zero indices"""
    rng = np.random.default_rng(c.seed + 77)
    c2r = c.transform == "r2c" and c.inverse
    reads = read_axes(c)
    ws, zs = [], []
    for a, n in enumerate(table_lengths(c)):
        if a not in reads:
            ws.append(np.full(n, complex(np.nan, np.nan), dtype=NPC[c.prec]))
            zs.append([])
            continue
        w = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        half = c.transform == "r2c" and a == 2
        if c2r:
            w = hermitian(w, half)
        z = zero_indices(n, c2r and not half)
        w[z] = 0
        ws.append(w.astype(NPC[c.prec]))
        zs.append(z)
    return ws, zs


def guarded(w, prec):
    """w on the device inside a buffer with GUARD NaN elements on each side (a view the plan reads)"""
    buf = torch.full((w.size + 2 * GUARD,), complex(math.nan, math.nan), dtype=TC[prec], device="cuda")
    buf[GUARD:GUARD + w.size] = torch.from_numpy(np.ascontiguousarray(w))
    return buf[GUARD:GUARD + w.size]


def spectral_shape(c):
    p = c.plan()
    k, m = table_lengths(c), c.data or c.shape
    reads = transformed(p, c.d)
    return tuple(k[a] if a in reads else m[a] for a in range(3))


def inputs(c):
    """(input fields, field scales, long-double reference without weights applied yet: None) of a case"""
    p = c.plan()
    data = c.data or c.shape
    r2c = c.transform == "r2c"
    off = c.seed % 4
    if not c.inverse:
        return mixed((3,) + data, 0, c.prec, not r2c, c.seed, off=off)
    if not r2c:
        return mixed((3,) + spectral_shape(c), 0, c.prec, True, c.seed, off=off)
    xr, sc = mixed((3,) + data, 0, c.prec, False, c.seed, off=off)
    x = np.stack([fwd_ref(p, (None, None, None), ld(xr[f]), c.d) for f in range(3)]).astype(NPC[c.prec])
    # an even K < N on x or y keeps -K/2 without +K/2: not the spectrum of a real field (test_gpu_accuracy family 2)
    spec_ = c.spectral or c.shape
    for a in (0, 1):
        if a in transformed(p, c.d) and spec_[a] < c.shape[a] and spec_[a] % 2 == 0:
            idx = [slice(None)] * 4
            idx[a + 1] = spec_[a] // 2
            x[tuple(idx)] = 0
    return x, sc


def reference(c, x, ws):
    """the long-double output of the case on the fields x with the tables ws (numpy, as the device holds them)"""
    p = c.plan()
    wl = tuple(ld(w) if c.weighted and a in read_axes(c) else None for a, w in enumerate(ws))
    if not c.inverse:
        return np.stack([fwd_ref(p, wl, ld(x[f]), c.d) for f in range(3)])
    ref = np.stack([inv_ref(p, wl, ld(x[f]), c.d) for f in range(3)])
    return ref.real if c.transform == "r2c" else ref


# ---- describe: the kernels a case launches -----------------------------------------------------------------------------
def twin_kinds(sc, prec, env):
    """{(precision, log2 n, kind)} of the weighted twins a step list launches, by the rules of launch_twin (TILED: wide
    when forced by DFFT_WIDE_TILES = 1, or automatic with rows >= 1 MiB apart from 1024 points on, and B > TBT) and
    launch_bluestein; the one-rank sequential schedule leaves the passes' tile preference automatic"""
    w = int(env) if env else 0
    esz = 16 if prec == F64 else 8
    out = set()
    for st in sc["steps"]:
        if st["type"] != 0 or "weighted" not in st:
            continue
        kind, lg = st["kind"], st["log2n"]
        if "n" in st:
            name = "Bluestein " + ("CONTIG" if kind == 0 else "TILED")
        elif kind == 0:
            name = "CONTIG"
        elif kind == 1:
            _, tbt, wide = shape_of(prec, lg)
            far = max(st["in"]["sN"], st["out"]["sN"]) * esz >= 1 << 20
            is_wide = wide != tbt and w >= 0 and st["B"] > tbt and (w > 0 or (w == 0 and lg >= 10 and far))
            name = "wide TILED" if is_wide else "TILED"
        elif kind == 2:
            name = "R2C"
        else:
            assert kind == 3, st
            name = "C2R shuffle" if lg - min(lg, 4) <= 5 else "C2R smem"  # TPL = M / 2^min(log2 M, 4) <= 32: one warp
        out.add((PIDS[PRECS.index(prec)], lg, name))
    return out


def required_kinds():
    need = set()
    for prec, pid in zip(PRECS, PIDS):
        for lg in range(1, 14):
            _, tbt, wide = shape_of(prec, lg)
            need |= {(pid, lg, "CONTIG"), (pid, lg, "TILED"), (pid, lg, "R2C"), (pid, lg, "C2R shuffle" if lg <= 9 else "C2R smem")}
            if wide != tbt:
                need.add((pid, lg, "wide TILED"))
        for n in BLUESTEIN:
            need |= {(pid, run_log2(n), "Bluestein CONTIG"), (pid, run_log2(n), "Bluestein TILED")}
    return need


def check_x_pass(c, sc):
    """the x pass runs B columns, B > TBT when the case forces wide tiles of a length whose widths differ"""
    if c.B is None:
        return
    xs = [st for st in sc["steps"] if st["type"] == 0 and st["label"] == "x pass"]
    assert xs and all(st["B"] == c.B for st in xs), f"{c.what()}: x pass B {[st['B'] for st in xs]}, wanted {c.B}"
    _, tbt, wide = shape_of(c.prec, xs[0]["log2n"])
    if c.env == "1" and wide != tbt:
        assert c.B > tbt, f"{c.what()}: B = {c.B} <= TBT = {tbt}: the wide run would run narrow tiles"


# ---- the GPU run ------------------------------------------------------------------------------------------------------------
def make_plan(c):
    kw = dict(batch=3)
    if c.spectral is not None:
        kw["spectral"] = c.spectral
    if c.data is not None:
        kw["data"] = c.data
    if c.axes is not None:
        kw["transform_axes"] = c.axes
    return plan_of(c.prec, c.transform, c.shape, **kw)


def execute(plan, c, out, inp):
    if c.transform == "c2c":
        plan.execC2C(out, inp, dfft.INVERSE if c.inverse else dfft.FORWARD, c.d)
    elif c.inverse:
        plan.execC2R(out, inp, c.d)
    else:
        plan.execR2C(out, inp, c.d)


def run_case(c, monkeypatch):
    if c.env is not None:
        monkeypatch.setenv("DFFT_WIDE_TILES", c.env)
    ws, zs = tables(c)
    x, sc = inputs(c)
    ref = reference(c, x, ws)
    real_out = c.transform == "r2c" and c.inverse
    out_shape, out_dt = ref.shape, TR[c.prec] if real_out else TC[c.prec]
    s = dict(spec(c.prec, c.shape, c.d), axes=c.axes or (1, 1, 1))
    plan = make_plan(c)
    plain = make_plan(c) if c.weighted else None
    try:
        assert tuple(plan.getPartialSize(c.d)) == (x.shape[1:] if c.inverse else ref.shape[1:]), c.what()
        assert not c.inverse or tuple(plan.getInSize()) == ref.shape[1:], c.what()
        if c.weighted:
            plan.setWeights(*[guarded(w, c.prec) for w in ws])
        sched = json.loads(R.describe_raw(plan._h, c.inverse, c.d))
        check_x_pass(c, sched)
        assert c.weighted == any("weighted" in st for st in sched["steps"]), c.what()
        fn = lambda o, i: execute(plan, c, o, i)  # noqa: E731
        got = on_device(fn, x, out_shape, out_dt)
        check_units(c.family, s, got, ref, 0, sc, c.what(), worst=WORST)
        if c.weighted and not c.inverse:
            for a, z in enumerate(zs):
                if z:
                    idx = [slice(None)] * 4
                    idx[a + 1] = z
                    assert not np.any(got[tuple(idx)]), f"{c.what()}: a zero weight of axis {a} gave a nonzero output"
        # the scale rule: the scaled exec is the scale-1 exec times s, rounded once in the plan's precision
        plan.setScale(SCALE, SCALE)
        got3 = on_device(fn, x, out_shape, out_dt)
        rt = NPR[c.prec]
        assert np.array_equal(got3.view(rt), got.view(rt) * rt(SCALE)), f"{c.what()}: the scaled exec is not the scale-1 exec times the scale"
        if c.scaled:
            check_units(c.family, s, got3, ref * exact_scale(c.prec, SCALE), 0, sc, c.what() + " scaled", worst=WORST)
        if c.weighted:
            # all-ones weights: the unweighted plan's values
            plan.setScale(1.0, 1.0)
            plan.setWeights(*[guarded(np.ones(w.size, dtype=NPC[c.prec]), c.prec) for w in ws])
            ones = on_device(fn, x, out_shape, out_dt)
            base = on_device(lambda o, i: execute(plain, c, o, i), x, out_shape, out_dt)
            assert np.array_equal(ones, base), f"{c.what()}: all-ones weights differ from the unweighted plan"
    finally:
        plan.destroy()
        if plain is not None:
            plain.destroy()


@pytest.mark.gpu
@pytest.mark.parametrize("transform,lg", Z_LENGTHS)
def test_weighted_z(transform, lg, monkeypatch):
    for c in w1_cases(transform, lg):
        run_case(c, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("env", ["1", "-1"])
@pytest.mark.parametrize("transform,lg", X_LENGTHS)
def test_weighted_x(transform, lg, env, monkeypatch):
    for c in w2_cases(transform, lg, env):
        run_case(c, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", [2, 0], ids=["z", "x"])
def test_weighted_bluestein(axis, monkeypatch):
    for c in w3_cases(axis):
        run_case(c, monkeypatch)


P1_SWEEPS = [(t, lg, 2) for t, lg in Z_LENGTHS] + [(t, lg, 0) for t, lg in X_LENGTHS]


@pytest.mark.gpu
@pytest.mark.parametrize("transform,lg,axis", P1_SWEEPS)
def test_pruned(transform, lg, axis, monkeypatch):
    for c in p1_cases(transform, lg, axis):
        run_case(c, monkeypatch)


# ---- CPU: the cases reach every weighted twin ----------------------------------------------------------------------------
def test_weighted_cases_launch_every_twin():
    got = set()
    for c in weighted_cases():
        sc = WR.describe(c.plan(), [np.ones(n) for n in table_lengths(c)], 0, c.inverse, c.d)
        check_x_pass(c, sc)
        got |= twin_kinds(sc, c.prec, c.env)
    missing = sorted(required_kinds() - got)
    assert not missing, f"weighted twins no case launches: {missing}"


def test_cases_keep_their_shapes():
    """every case fits CAP; the pruned and padded ones have the holes they were made for"""
    for c in weighted_cases() + [c for t, lg, a in P1_SWEEPS for c in p1_cases(t, lg, a)]:
        assert 3 * math.prod(c.shape) <= CAP, c.what()
        sc = R.describe(c.plan(), 0, c.inverse, c.d)
        check_x_pass(c, sc)
        assert ("data" in sc) == (c.data is not None) and ("spectral" in sc) == (c.spectral is not None), c.what()


# ---- CPU: the reference --------------------------------------------------------------------------------------------------
def dense_reference(c, x, ws):
    """the case's output by dense DFT matrices in long double, one axis at a time: an independent definition of the zero
    embedding, the truncation to K, the weights and the data block"""
    p = c.plan()
    data, spec_ = c.data or c.shape, c.spectral or c.shape
    reads = read_axes(c)
    two_pi = 2 * np.arccos(np.longdouble(-1))  # pi in long double
    out = ld(x)
    for a in ((2, 1, 0) if not c.inverse else (0, 1, 2)):
        if a not in reads:
            continue
        n, half = c.shape[a], c.transform == "r2c" and a == 2
        freq = R.positions(n, spec_[a], half).astype(np.longdouble)
        w = ld(ws[a]) if c.weighted else np.ones(freq.size, dtype=np.clongdouble)
        pos = np.arange(data[a], dtype=np.longdouble)
        if not c.inverse:
            mat = np.exp(-1j * two_pi * np.outer(freq, pos) / n) * w[:, None]  # [k, m]
            out = np.moveaxis(np.tensordot(mat, out, axes=([1], [a + 1])), 0, a + 1)
        else:
            mat = np.exp(1j * two_pi * np.outer(pos, freq) / n) * w[None, :]  # [m, k]
            if half:  # the real line of a half spectrum: X_0 and X_{N/2} count once, every other mode with its conjugate
                mult = np.where((freq == 0) | (2 * freq == n), 1, 2).astype(np.longdouble)
                y = np.tensordot(mat.real * mult[None, :], out.real, axes=([1], [a + 1])) - np.tensordot(mat.imag * mult[None, :], out.imag, axes=([1], [a + 1]))
                out = np.moveaxis(y, 0, a + 1)
            else:
                out = np.moveaxis(np.tensordot(mat, out, axes=([1], [a + 1])), 0, a + 1)
    return out.real if c.transform == "r2c" and c.inverse else out


def small_cases():
    out = [c for t, lg in (("c2c", 2), ("c2c", 4), ("r2c", 3), ("r2c", 4)) for c in w1_cases(t, lg)]
    out += [c for t, lg in (("c2c", 3), ("r2c", 2)) for env in ("1", "-1") for c in w2_cases(t, lg, env)]
    out += [c for c in w3_cases(2) + w3_cases(0) if max(c.shape) <= 9]
    return out + [c for t, lg in (("c2c", 4), ("r2c", 4)) for a in (2, 0) for c in p1_cases(t, lg, a)]


def test_reference_against_dense_dft_and_double():
    """the long-double reference equals dense DFT matrices, and test_weights.fwd_ref / inv_ref in double"""
    for c in small_cases():
        ws, _ = tables(c)
        x, _ = inputs(c)
        ref = reference(c, x, ws)
        assert ref.dtype == (np.longdouble if c.transform == "r2c" and c.inverse else np.clongdouble), c.what()
        dense = dense_reference(c, x, ws)
        assert ref.shape == dense.shape, c.what()
        assert np.max(np.abs(ref - dense)) <= 1e-15 * np.max(np.abs(dense)), c.what()
        p = c.plan()
        wd = tuple(w.astype(np.complex128) if c.weighted and a in read_axes(c) else None for a, w in enumerate(ws))
        if c.inverse:
            dbl = np.stack([inv_ref(p, wd, x[f].astype(np.complex128), c.d) for f in range(3)])
            dbl = dbl.real if c.transform == "r2c" else dbl
        else:
            dbl = np.stack([fwd_ref(p, wd, x[f].astype(np.complex128 if c.transform == "c2c" else np.float64), c.d) for f in range(3)])
        assert dbl.dtype in (np.complex128, np.float64)
        assert np.max(np.abs(ref - dbl)) <= 1e-13 * np.max(np.abs(dense)), c.what()


def test_inverse_references_keep_long_double():
    import test_gpu_weights
    import test_pruned

    p = R.Plan(1, dfft.SLAB_ZY_THEN_X, (4, 4, 8), transform=dfft.R2C, spectral=(3, 4, 6), data=(2, 3, 6))
    X = np.ones((3, 4, 4), dtype=np.clongdouble)
    assert inv_ref(p, (None, None, None), X, 3).dtype == np.longdouble
    assert test_pruned.inv_ref(X, dfft.R2C, (4, 4, 8), (2, 3, 6), (3, 4, 6), 3).dtype == np.longdouble
    q = R.Plan(1, dfft.SLAB_ZY_THEN_X, (4, 4, 8), spectral=(3, 4, 6))
    assert inv_ref(q, (None, None, None), np.ones((3, 4, 6), dtype=np.clongdouble), 3).dtype == np.clongdouble
    case = test_gpu_weights.Case.__new__(test_gpu_weights.Case)
    case.batch, case.c2c, case.shape, case.spec, case.data = 1, False, (4, 4, 8), (3, 4, 6), (2, 3, 6)
    assert case.inverse_ref(X[None]).dtype == np.longdouble
    case.c2c = True
    assert case.inverse_ref(np.ones((1, 3, 4, 6), dtype=np.clongdouble)).dtype == np.clongdouble


# ---- CPU: plausible defects fail the per-field bound ---------------------------------------------------------------------
DEFECT_LENGTHS = (16, 256, 4096)


def worst_unit(s, got, ref, scales):
    errs = [error_check(s, got[i], ref[i]) for i in range(ref.shape[0]) if scales[i] != 0]
    return max(e[0] for e in errs), max(e[1] for e in errs)


def passes_bound(s, got, ref, scales):
    rel, mx = worst_unit(s, got, ref, scales)
    return rel <= REL_BOUND and mx <= MAX_BOUND


def half_weights(m, seed):
    rng = np.random.default_rng(seed)
    w = hermitian(rng.standard_normal(m + 1) + 1j * rng.standard_normal(m + 1), True)
    w[zero_indices(m + 1, False)] = 0
    return w


def c2r_emulation(X, w, prec, defect=None):
    """the weighted C2R pass in the plan's precision: X[k] w[k], then the unnormalised inverse; defect "partner": the
    partner X[M - k] of k <= M/2 weighted by w[k]; "nyquist": X[M] left unweighted"""
    m = X.shape[-1] - 1
    idx = np.arange(m + 1)
    if defect == "partner":
        idx[m // 2 + 1:] = m - idx[m // 2 + 1:]
    Y = X.astype(NPC[prec]) * w.astype(NPC[prec])[idx]
    if defect == "nyquist":
        Y[..., m] = X[..., m]
    return np.fft.irfft(Y, n=2 * m, axis=-1) * NPR[prec](2 * m)


@pytest.mark.parametrize("defect", ["partner", "nyquist"])
@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_c2r_weight_defects_fail_the_bound(prec, defect):
    for n in DEFECT_LENGTHS:
        m = n // 2
        xr, sc = mixed((8, n), 0, prec, False, n + 1)
        X = np.fft.rfft(ld(xr), axis=1).astype(NPC[prec])
        w = half_weights(m, n).astype(NPC[prec])
        ref = np.fft.irfft(ld(X) * ld(w), n=n, axis=1) * n
        s = spec(prec, (1, 1, n), 1)
        assert passes_bound(s, c2r_emulation(X, w, prec), ref, sc), (n, "the correct mapping")
        assert not passes_bound(s, c2r_emulation(X, w, prec, defect), ref, sc), (n, defect)


@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_padded_negative_block_off_by_one_fails_the_bound(prec):
    """a padded C2C forward whose negative-frequency block takes the weight one index too low"""
    for n in DEFECT_LENGTHS:
        x, sc = mixed((8, n), 0, prec, True, n + 2)
        for k in (n // 2 + 1, n - 1):
            rng = np.random.default_rng(k)
            w = (rng.standard_normal(k) + 1j * rng.standard_normal(k)).astype(NPC[prec])
            pos = R.positions(n, k)
            ref = np.fft.fft(ld(x), axis=1)[:, pos] * ld(w)
            X = np.fft.fft(x, axis=1)[:, pos]
            s = spec(prec, (1, 1, n), 1)
            assert passes_bound(s, X * w, ref, sc), (n, k)
            shifted = w.copy()
            shifted[(k + 1) // 2:] = w[(k + 1) // 2 - 1:-1]
            assert not passes_bound(s, X * shifted, ref, sc), (n, k)


@pytest.mark.parametrize("prec", PRECS, ids=PIDS)
def test_pruned_r2c_dropped_pair_fails_the_bound(prec):
    """a pruned R2C forward that reads its last data pair as zero"""
    for n in DEFECT_LENGTHS:
        for m in (n // 2, n - 2):
            xr, sc = mixed((8, m), 0, prec, False, n + m)
            ref = np.fft.rfft(ld(xr), n=n, axis=1)
            s = spec(prec, (1, 1, n), 1)
            assert passes_bound(s, np.fft.rfft(xr, n=n, axis=1), ref, sc), (n, m)
            dropped = xr.copy()
            dropped[:, m - 2:] = 0
            assert not passes_bound(s, np.fft.rfft(dropped, n=n, axis=1), ref, sc), (n, m)
