"""Type-I real-to-real kinds (DFFT_DCT1 / DFFT_DST1: DCT-I and DST-I) without a GPU.

- The type-I pass's per-line steps on the CPU (tests/emu_r2r1.cpp: r2r.hpp and fft_core.cuh's stage arithmetic) against a
  naive long-double DCT-I / DST-I for every N = 2..8192 (DST-I from 4), f64 and f32, and a zero line.
- Kind and length validation (5 and 7 still refused, dfft_plan_create* refuse 16 / 17, padded and interleaved plans refuse
  them as before), dfft_plan_get_r2r_kinds, and dfft_plan_describe: "dct1" / "dst1" in "r2r_kinds" and on the passes,
  "n" = L and "log2n" = log2 N on type-I passes, the sequential schedule also with send_method Streams.
- Lock-step replays of every rank's step list with scipy's dct / dst (type=1 on type-I passes) per pass, checked against
  the per-axis transform of the global array: 1-8 ranks, slab, Z_Then_YX and pencil, Peer2Peer and All2All, both
  directions, partial d, uneven splits, blocked layouts with tails, type-I / type-II / R2HC mixes, kept axes, batches,
  in-place plans and output scales (applied exactly once), with the happens-before check of every access
  (step_replay.py)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.fft as sf

import distributedfft_b200 as dfft
from distributedfft_b200._lib import check, lib
import step_replay as R
from test_r2r import CASES
from test_r2r_mixed import create_plain, create_r2r, destroy, hc2r, r2hc

HERE = os.path.dirname(os.path.abspath(__file__))
SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
DCT, DST, R2HC, DCT1, DST1 = dfft.DCT, dfft.DST, dfft.R2HC, dfft.DCT1, dfft.DST1
NAMES = {DCT: "dct", DST: "dst", R2HC: "r2hc", DCT1: "dct1", DST1: "dst1"}


def test_r2r1_kernel_math_matches_naive():
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "emu")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "emu_r2r1.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        print(r.stdout[-400:])
        assert r.returncode == 0, r.stdout[-2000:]
        assert "fails=0" in r.stdout


def axis_len(n, kind):
    """the length of an axis of kind `kind` built on the power of two n: n + 1 (DCT-I), n - 1 (DST-I), n otherwise"""
    return n + 1 if kind == DCT1 else n - 1 if kind == DST1 else n


def shape_for(base, kinds):
    return tuple(axis_len(n, k) for n, k in zip(base, kinds))


# ---- references ------------------------------------------------------------------------------------------------------
def r2r_1d(x, kind, inverse, axis):
    if kind == R2HC:
        return hc2r(x, axis) if inverse else r2hc(x, axis)
    if kind in (DCT1, DST1):  # its own inverse up to 2N: both directions run it
        return (sf.dct if kind == DCT1 else sf.dst)(x, type=1, axis=axis)
    return (sf.dct if kind == DCT else sf.dst)(x, type=3 if inverse else 2, axis=axis)


def global_ref(x, kinds, inverse, d, taxes=(1, 1, 1)):
    """the first d axes in z, y, x order, each with its kind; kept axes untouched"""
    for axis in (2, 1, 0)[:d]:
        if taxes[axis]:
            x = r2r_1d(x, kinds[axis], inverse, axis)
    return x


def test_type1_references_are_their_own_inverse():
    rng = np.random.default_rng(3)
    for n in (2, 4, 64):
        x = rng.standard_normal(n + 1)
        assert np.allclose(sf.dct(sf.dct(x, type=1), type=1), 2 * n * x)
        if n >= 4:
            x = rng.standard_normal(n - 1)
            assert np.allclose(sf.dst(sf.dst(x, type=1), type=1), 2 * n * x)


# ---- validation ------------------------------------------------------------------------------------------------------
def test_kind_validation():
    for kinds in ((DCT1, DST1, R2HC), (DST1, DST1, DST1), (DCT1, DCT, DST)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, shape_for((8, 8, 8), kinds), 1, 1)
        assert rc == 0, kinds
        destroy(c, plan)
    for kinds in ((2, 2, 5), (3, 7, 4), (15, 2, 2), (18, 2, 2), (16, 16, 8), (16, 17, -1)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, (9, 9, 9), 1, 1)
        assert rc == -1, kinds  # DFFT_ERR_INVALID
        destroy(c, plan)
    # a plan's kinds come only through dfft_plan_create_r2r: 16 / 17 are no plan transform, like 4
    for transform in (4, 5, 7, 16, 17):
        for inplace in (False, True):
            rc, c, plan = create_plain(0, 1, SL, transform, (9, 9, 9), 1, 1, inplace=inplace)
            assert rc == -1, (transform, inplace)
            destroy(c, plan)
    for t in (0, 1, 5, 7, 15, 18):
        assert lib().dfft_fft1d_r2r(dfft.F64, t, -1, 9, 1, 1, None, None, None) == -1


def test_padded_and_interleaved_plans_refuse_type1():
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(0, 1, C.byref(c)))
    plan = C.c_void_p()
    for t in (DCT1, DST1):
        assert lib().dfft_plan_create_padded(c, None, SL, dfft.F64, t, 9, 9, 9, 9, 9, 9, 1, 1, 1, 1, C.byref(plan)) == -1
        for comps in (1, 3):
            assert lib().dfft_plan_create_interleaved(c, None, SL, dfft.F64, t, 9, 9, 9, 1, 1, comps, 1, 1, C.byref(plan)) == -1
    lib().dfft_comm_destroy(c)


def dct1_ok(n):
    return n >= 3 and (n - 1) & (n - 2) == 0 and n - 1 <= 8192


def dst1_ok(n):
    return n >= 3 and (n + 1) & n == 0 and n + 1 <= 8192


@pytest.mark.parametrize("kind", [DCT1, DST1])
def test_length_validation(kind):
    good = dct1_ok if kind == DCT1 else dst1_ok
    lengths = list(range(0, 70)) + [127, 128, 129, 255, 256, 257, 4095, 4096, 4097, 8191, 8192, 8193, 8194, 16383, 16384, 16385]
    for n in lengths:
        for axis in range(3):
            kinds = [DCT] * 3
            kinds[axis] = kind
            shape = [4, 4, 4]
            shape[axis] = n
            rc, c, plan = create_r2r(0, 1, SL, tuple(kinds), tuple(shape), 1, 1)
            want = 0 if good(n) else (-1 if n == 0 else -5)  # n == 0 is no grid at all
            assert rc == want, (kind, axis, n, rc)
            destroy(c, plan)
        # the single-axis call: validated before anything runs (a = 0 lines then returns at once)
        assert lib().dfft_fft1d_r2r(dfft.F64, kind, -1, n, 0, 1, None, None, None) == (0 if good(n) else -5), n


def test_kept_axis_keeps_its_kinds_length_rule():
    """a kept type-I axis still needs a length its kind takes: the kinds are checked when the plan is created"""
    rc, c, plan = create_r2r(0, 1, SL, (DCT1, R2HC, R2HC), (16, 8, 8), 1, 1)
    assert rc == -5
    destroy(c, plan)
    rc, c, plan = create_r2r(0, 1, SL, (DCT1, R2HC, R2HC), (17, 8, 8), 1, 1)
    assert rc == 0
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == 0
    destroy(c, plan)


def test_get_r2r_kinds():
    k = (C.c_int * 3)()
    for kinds in ((DCT1, R2HC, R2HC), (DST1, DST1, DST1), (DCT1, DST, DST1), (R2HC, DCT1, DCT)):
        rc, c, plan = create_r2r(0, 4, PE, kinds, shape_for((8, 16, 32), kinds), 2, 2)
        assert rc == 0
        check(lib().dfft_plan_get_r2r_kinds(plan, k))
        assert tuple(k) == kinds
        destroy(c, plan)


def plan_of(P, decomp, kinds, shape, p1, p2, comm, send, batch=1, prec=dfft.F64, scale=None, inplace=False, taxes=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, kinds=kinds, prec=prec, comm=comm, send=send, batch=batch, inplace=inplace, scale=scale, axes=taxes)


def describe(rank, P, decomp, kinds, shape, p1, p2, comm, send, inverse, d, batch=1, prec=dfft.F64, scale=None, inplace=False, taxes=None):
    return R.describe(plan_of(P, decomp, kinds, shape, p1, p2, comm, send, batch, prec, scale, inplace, taxes), rank, inverse, d)


@pytest.mark.parametrize("kinds", [(DCT1, R2HC, R2HC), (DST1, DST1, DST1), (DCT1, DST, DST1), (DCT1, DCT1, DCT1)],
                         ids=lambda k: "-".join(NAMES[x] for x in k))
def test_describe(kinds):
    shape = shape_for((16, 32, 64), kinds)
    for P, decomp, p1, p2 in ((1, SL, 1, 1), (4, ZY, 4, 1), (4, PE, 2, 2)):
        for send in (SYNC, STREAMS):  # Streams plans run the sequential schedule
            for inverse in (0, 1):
                sc = describe(0, P, decomp, kinds, shape, p1, p2, P2P, send, inverse, 3)
                assert sc["r2r_kinds"] == [NAMES[k] for k in kinds]
                assert sc["r2r"] == (NAMES[kinds[0]] if len(set(kinds)) == 1 else "mixed")
                assert not sc["overlapped"] and all(s["stream"] == 0 for s in sc["steps"])
                passes = [s for s in sc["steps"] if s["type"] == 0]
                assert {s["kind"] for s in passes} <= {4, 5}
                for s in passes:
                    if s["r2r"] in ("dct1", "dst1"):
                        n = s["n"]
                        assert n == (1 << s["log2n"]) + (1 if s["r2r"] == "dct1" else -1)
                    else:
                        assert "n" not in s
                z = passes[-1 if inverse else 0]
                assert z["kind"] == 4 and z["r2r"] == NAMES[kinds[2]] and z.get("n", 1 << z["log2n"]) == shape[2]


# ---- lock-step replay ---------------------------------------------------------------------------------------------------
def run_type1(P, decomp, kinds, shape, p1, p2, comm, send, inverse, d, batch=1, inplace=False, scale=None, prec=dfft.F64, taxes=None):
    """replays every rank's steps in lock step, each pass with the kind its description names and the length "n" of
    type-I passes; returns the worst rel-L2 error of any rank's output block against the per-axis global transform, and
    whether a type-I pass ran"""
    nx, ny, nz = shape
    p = plan_of(P, decomp, kinds, shape, p1, p2, comm, send, batch, prec, scale, inplace, taxes)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    assert not scheds[0]["overlapped"]
    ta = taxes or (1, 1, 1)
    rng = np.random.default_rng(P * 1000 + nx + ny + nz + batch + 7 * kinds[0] + 3 * kinds[1] + kinds[2])
    xg = rng.standard_normal((batch,) + shape)
    spec = np.stack([global_ref(xg[f], kinds, False, d, ta) for f in range(batch)])
    want_g = np.stack([global_ref(spec[f], kinds, True, d, ta) for f in range(batch)]) if inverse else spec
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    if prec == dfft.F32:
        s_used = float(np.float32(s_used))
    worst = R.error(R.replay(p, inverse, d, spec if inverse else xg, scheds), want_g * s_used)
    seen_type1 = any(st.get("r2r") in ("dct1", "dst1") for sc in scheds for st in sc["steps"] if st["type"] == 0)
    return worst, seen_type1


def replay(P, decomp, kinds, base, p1, p2, comm, send, inverse, d, **kw):
    worst, seen = run_type1(P, decomp, kinds, shape_for(base, kinds), p1, p2, comm, send, inverse, d, **kw)
    assert seen or d < 3, "no type-I pass ran"
    return worst


MIXES = [(DCT1, DCT1, DCT1), (DST1, DST1, DST1), (DCT1, R2HC, R2HC), (DST1, DCT, DCT1), (R2HC, DST1, DST), (DCT1, DST1, R2HC)]


@pytest.mark.parametrize("kinds", MIXES, ids=lambda k: "-".join(NAMES[x] for x in k))
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", CASES)
def test_replay_full(P, decomp, shape, p1, p2, comm, send, inverse, kinds):
    """test_r2r's 1-8 rank cases with every axis of length 2^k +- 1: uneven splits on every rank count, blocked tails"""
    assert replay(P, decomp, kinds, shape, p1, p2, comm, send, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_replay_partial(d, inverse, comm):
    assert replay(8, PE, (DCT1, R2HC, DST1), (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert replay(6, PE, (DCT, DST1, DCT1), (8, 16, 16), 2, 3, comm, SYNC, inverse, d) < 1e-12
    assert replay(3, SL, (R2HC, DCT1, DST1), (8, 16, 64), 3, 1, comm, SYNC, inverse, d) < 1e-12
    assert replay(1, SL, (DST1, DCT1, DCT1), (8, 4, 16), 1, 1, comm, SYNC, inverse, d) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("kinds", [(DCT1, R2HC, R2HC), (DST1, DST1, DST1), (DCT1, DST, DST1)], ids=lambda k: "-".join(NAMES[x] for x in k))
def test_replay_batch_inplace_scale(kinds, inverse):
    s = (0.25, 1.0 / 3.0)
    assert replay(1, SL, kinds, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, batch=3) < 1e-12
    assert replay(3, SL, kinds, (8, 16, 64), 3, 1, P2P, SYNC, inverse, 3, batch=3, scale=s) < 1e-12
    assert replay(1, SL, kinds, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, inplace=True, scale=s) < 1e-12
    assert replay(1, PE, kinds, (8, 16, 32), 1, 1, P2P, SYNC, inverse, 2, inplace=True, batch=3) < 1e-12
    assert replay(4, PE, kinds, (8, 16, 32), 2, 2, A2A, SYNC, inverse, 3, inplace=True, batch=3, scale=s) < 1e-12
    assert replay(3, ZY, kinds, (8, 4, 16), 3, 1, P2P, SYNC, inverse, 3, inplace=True, scale=s, prec=dfft.F32) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("taxes", [(0, 1, 1), (1, 0, 1), (1, 1, 0)])
def test_replay_kept_axes(taxes, inverse):
    """a kept type-I axis is moved by the copy pass like any kept axis"""
    s = (0.5, 2.0)
    for kinds in ((DCT1, R2HC, DST1), (DST1, DCT1, DCT)):
        assert replay(1, SL, kinds, (8, 16, 32), 1, 1, P2P, SYNC, inverse, 3, taxes=taxes) < 1e-12
        assert replay(4, PE, kinds, (8, 16, 32), 2, 2, A2A, SYNC, inverse, 3, taxes=taxes, scale=s) < 1e-12
        assert replay(3, ZY, kinds, (8, 4, 16), 3, 1, P2P, SYNC, inverse, 3, taxes=taxes, batch=3) < 1e-12


def test_blocked_slab_hand_over_with_tail():
    """a one-rank and a two-rank slab plan large enough for the blocked y -> x hand-over, its Nz % CH tail included"""
    kinds = (DCT1, DST1, DCT1)
    for P in (1, 2):
        sc = describe(0, P, SL, kinds, (257, 255, 257), P, 1, P2P, SYNC, 0, 3)
        x = [s for s in sc["steps"] if s["type"] == 0 and s["label"].startswith("x")]
        assert x and x[0]["B"] < 255 * 257, "not the blocked layout"
    for inverse in (0, 1):
        assert run_type1(2, SL, kinds, (257, 255, 257), 2, 1, P2P, SYNC, inverse, 3)[0] < 1e-12
