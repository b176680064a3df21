"""Type-IV real-to-real kinds (DFFT_DCT4 / DFFT_DST4: DCT-IV and DST-IV) without a GPU.

- The type-IV pass's per-line steps on the CPU (tests/emu_r2r4.cpp: r2r.hpp's helpers and host table, fft_core.cuh's stage
  arithmetic) against a naive long-double DCT-IV / DST-IV for every N = 4..8192, f64 and f32, and a zero line.
- Kind and length validation (18 still refused, dfft_plan_create* refuse 19 / 20, padded and interleaved plans refuse them
  as every R2R transform), dfft_plan_get_r2r_kinds, the Python names, and dfft_plan_describe: "dct4" / "dst4" in
  "r2r_kinds" and on the passes, "log2n" = log2 N and no "n" on type-IV passes, the sequential schedule also with
  send_method Streams.
- Lock-step replays of every rank's step list with scipy's dct / dst (type=4 on type-IV passes) per pass, checked against
  the per-axis transform of the global array: 1-8 ranks, slab, Z_Then_YX and pencil, Peer2Peer and All2All, both
  directions, partial d, uneven splits, blocked layouts with tails, type-IV / type-I / type-II / R2HC mixes, kept axes,
  batches, in-place plans and output scales (applied exactly once), with the happens-before check of every access
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
from test_r2r1 import axis_len, r2r_1d as r2r_1d_type1
from test_r2r_mixed import create_plain, create_r2r, destroy

HERE = os.path.dirname(os.path.abspath(__file__))
SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
DCT, DST, R2HC, DCT1, DST1, DCT4, DST4 = dfft.DCT, dfft.DST, dfft.R2HC, dfft.DCT1, dfft.DST1, dfft.DCT4, dfft.DST4
NAMES = {DCT: "dct", DST: "dst", R2HC: "r2hc", DCT1: "dct1", DST1: "dst1", DCT4: "dct4", DST4: "dst4"}

# the replay engine's pass math for type-IV passes: its own inverse up to 2N, so both directions run it
R.R2R.setdefault("dct4", lambda x, inv: sf.dct(x, type=4, axis=2))
R.R2R.setdefault("dst4", lambda x, inv: sf.dst(x, type=4, axis=2))


def test_r2r4_kernel_math_matches_naive():
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "emu")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "emu_r2r4.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        print(r.stdout[-400:])
        assert r.returncode == 0, r.stdout[-2000:]
        assert "fails=0" in r.stdout


def shape_for(base, kinds):
    """type-IV axes take the power of two itself, type-I ones 2^k +- 1"""
    return tuple(axis_len(n, k) for n, k in zip(base, kinds))


# ---- references ------------------------------------------------------------------------------------------------------
def r2r_1d(x, kind, inverse, axis):
    if kind in (DCT4, DST4):
        return (sf.dct if kind == DCT4 else sf.dst)(x, type=4, axis=axis)
    return r2r_1d_type1(x, kind, inverse, axis)


def global_ref(x, kinds, inverse, d, taxes=(1, 1, 1)):
    """the first d axes in z, y, x order, each with its kind; kept axes untouched"""
    for axis in (2, 1, 0)[:d]:
        if taxes[axis]:
            x = r2r_1d(x, kinds[axis], inverse, axis)
    return x


def test_type4_references_are_their_own_inverse():
    rng = np.random.default_rng(3)
    for n in (4, 8, 64):
        x = rng.standard_normal(n)
        assert np.allclose(sf.dct(sf.dct(x, type=4), type=4), 2 * n * x)
        assert np.allclose(sf.dst(sf.dst(x, type=4), type=4), 2 * n * x)


# ---- validation ------------------------------------------------------------------------------------------------------
def test_kind_validation():
    for kinds in ((DCT4, DST4, R2HC), (DST4, DST4, DST4), (DCT4, DCT, DST), (DCT1, DCT4, DST1), (DCT4, DCT4, DCT4)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, shape_for((8, 8, 8), kinds), 1, 1)
        assert rc == 0, kinds
        destroy(c, plan)
    for kinds in ((18, 2, 2), (19, 21, 4), (2, 18, 20), (20, 19, -1)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, (8, 8, 8), 1, 1)
        assert rc == -1, kinds  # DFFT_ERR_INVALID
        destroy(c, plan)
    # a plan's kinds come only through dfft_plan_create_r2r: 19 / 20 are no plan transform, like 4, 16 and 17
    for transform in (18, 19, 20):
        for inplace in (False, True):
            rc, c, plan = create_plain(0, 1, SL, transform, (8, 8, 8), 1, 1, inplace=inplace)
            assert rc == -1, (transform, inplace)
            destroy(c, plan)
    for t in (18, 21):
        assert lib().dfft_fft1d_r2r(dfft.F64, t, -1, 8, 1, 1, None, None, None) == -1
    for t in (DCT4, DST4):
        assert lib().dfft_fft1d_r2r(dfft.F64, t, -1, 8, 0, 1, None, None, None) == 0


def test_padded_and_interleaved_plans_refuse_type4():
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(0, 1, C.byref(c)))
    plan = C.c_void_p()
    for t in (DCT4, DST4):
        assert lib().dfft_plan_create_padded(c, None, SL, dfft.F64, t, 8, 8, 8, 8, 8, 8, 1, 1, 1, 1, C.byref(plan)) == -1
        for comps in (1, 3):
            assert lib().dfft_plan_create_interleaved(c, None, SL, dfft.F64, t, 8, 8, 8, 1, 1, comps, 1, 1, C.byref(plan)) == -1
    lib().dfft_comm_destroy(c)


def type4_ok(n):
    return 4 <= n <= 8192 and n & (n - 1) == 0


@pytest.mark.parametrize("kind", [DCT4, DST4])
def test_length_validation(kind):
    lengths = list(range(0, 70)) + [127, 128, 129, 255, 256, 257, 4095, 4096, 4097, 8191, 8192, 8193, 16384]
    for n in (2, 3, 6, 12, 16384):
        assert not type4_ok(n)
    assert type4_ok(4) and type4_ok(8192)
    for n in lengths:
        for axis in range(3):
            kinds = [DCT] * 3
            kinds[axis] = kind
            shape = [4, 4, 4]
            shape[axis] = n
            rc, c, plan = create_r2r(0, 1, SL, tuple(kinds), tuple(shape), 1, 1)
            want = 0 if type4_ok(n) else (-1 if n == 0 else -5)  # n == 0 is no grid at all
            assert rc == want, (kind, axis, n, rc)
            destroy(c, plan)
        # the single-axis call: validated before anything runs (a = 0 lines then returns at once)
        assert lib().dfft_fft1d_r2r(dfft.F64, kind, -1, n, 0, 1, None, None, None) == (0 if type4_ok(n) else -5), n


def test_kept_axis_keeps_its_kinds_length_rule():
    """a kept type-IV axis still needs a length its kind takes: the kinds are checked when the plan is created"""
    rc, c, plan = create_r2r(0, 1, SL, (DCT4, R2HC, R2HC), (2, 8, 8), 1, 1)
    assert rc == -5
    destroy(c, plan)
    rc, c, plan = create_r2r(0, 1, SL, (DST4, R2HC, R2HC), (16, 8, 8), 1, 1)
    assert rc == 0
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == 0
    destroy(c, plan)


def test_get_r2r_kinds():
    k = (C.c_int * 3)()
    for kinds in ((DCT4, R2HC, R2HC), (DST4, DST4, DST4), (DCT4, DST, DST1), (R2HC, DCT1, DST4)):
        rc, c, plan = create_r2r(0, 4, PE, kinds, shape_for((8, 16, 32), kinds), 2, 2)
        assert rc == 0
        check(lib().dfft_plan_get_r2r_kinds(plan, k))
        assert tuple(k) == kinds
        destroy(c, plan)


def test_python_names():
    assert (dfft.DCT4, dfft.DST4) == (19, 20)
    f = dfft.MPIcuFFT(None, comm=object(), transform=("dct4", "R2HC", "dst4"))
    assert f.kinds == (DCT4, R2HC, DST4) and f.transform == R2HC
    f = dfft.MPIcuFFT(None, comm=object(), transform=("dct4", "dct4", "dct4"))
    assert f.kinds == (DCT4,) * 3 and f.transform == R2HC  # a per-axis plan, like type I
    with pytest.raises(ValueError):
        dfft.MPIcuFFT(None, comm=object(), transform=("dct4", "dct3", "r2hc"))


def plan_of(P, decomp, kinds, shape, p1, p2, comm, send, batch=1, prec=dfft.F64, scale=None, inplace=False, taxes=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, kinds=kinds, prec=prec, comm=comm, send=send, batch=batch, inplace=inplace, scale=scale, axes=taxes)


def describe(rank, P, decomp, kinds, shape, p1, p2, comm, send, inverse, d, batch=1, prec=dfft.F64, scale=None, inplace=False, taxes=None):
    return R.describe(plan_of(P, decomp, kinds, shape, p1, p2, comm, send, batch, prec, scale, inplace, taxes), rank, inverse, d)


@pytest.mark.parametrize("kinds", [(DCT4, R2HC, R2HC), (DST4, DST4, DST4), (DCT4, DST, DST1), (DCT4, DCT4, DCT4), (DCT1, DST4, DCT4)],
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
                seen = set()
                for s in passes:
                    if s["r2r"] in ("dct4", "dst4"):  # log2n = log2 N, the line length: no "n"
                        assert "n" not in s and (1 << s["log2n"]) in shape
                        seen.add(s["r2r"])
                assert seen == {NAMES[k] for k in kinds if k in (DCT4, DST4)}
                z = passes[-1 if inverse else 0]
                assert z["kind"] == 4 and z["r2r"] == NAMES[kinds[2]] and z.get("n", 1 << z["log2n"]) == shape[2]


# ---- lock-step replay ---------------------------------------------------------------------------------------------------
def run_type4(P, decomp, kinds, shape, p1, p2, comm, send, inverse, d, batch=1, inplace=False, scale=None, prec=dfft.F64, taxes=None):
    """replays every rank's steps in lock step, each pass with the kind its description names; returns the worst rel-L2
    error of any rank's output block against the per-axis global transform, and whether a type-IV pass ran"""
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
    seen = any(st.get("r2r") in ("dct4", "dst4") for sc in scheds for st in sc["steps"] if st["type"] == 0)
    return worst, seen


def replay(P, decomp, kinds, base, p1, p2, comm, send, inverse, d, **kw):
    worst, seen = run_type4(P, decomp, kinds, shape_for(base, kinds), p1, p2, comm, send, inverse, d, **kw)
    assert seen or d < 3, "no type-IV pass ran"
    return worst


MIXES = [(DCT4, DCT4, DCT4), (DST4, DST4, DST4), (DCT4, R2HC, R2HC), (DST4, DCT, DCT4), (R2HC, DST4, DST), (DCT4, DST1, R2HC),
         (DCT1, DCT4, DST4)]


@pytest.mark.parametrize("kinds", MIXES, ids=lambda k: "-".join(NAMES[x] for x in k))
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", CASES)
def test_replay_full(P, decomp, shape, p1, p2, comm, send, inverse, kinds):
    """test_r2r's 1-8 rank cases: uneven splits on every rank count, blocked tails"""
    assert replay(P, decomp, kinds, shape, p1, p2, comm, send, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_replay_partial(d, inverse, comm):
    assert replay(8, PE, (DCT4, R2HC, DST4), (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert replay(6, PE, (DCT, DST4, DCT4), (8, 16, 16), 2, 3, comm, SYNC, inverse, d) < 1e-12
    assert replay(3, SL, (R2HC, DCT4, DST1), (8, 16, 64), 3, 1, comm, SYNC, inverse, d) < 1e-12
    assert replay(1, SL, (DST4, DCT1, DCT4), (8, 4, 16), 1, 1, comm, SYNC, inverse, d) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("kinds", [(DCT4, R2HC, R2HC), (DST4, DST4, DST4), (DCT4, DST, DST1)], ids=lambda k: "-".join(NAMES[x] for x in k))
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
    """a kept type-IV axis is moved by the copy pass like any kept axis"""
    s = (0.5, 2.0)
    for kinds in ((DCT4, R2HC, DST4), (DST4, DCT4, DCT1)):
        assert replay(1, SL, kinds, (8, 16, 32), 1, 1, P2P, SYNC, inverse, 3, taxes=taxes) < 1e-12
        assert replay(4, PE, kinds, (8, 16, 32), 2, 2, A2A, SYNC, inverse, 3, taxes=taxes, scale=s) < 1e-12
        assert replay(3, ZY, kinds, (8, 4, 16), 3, 1, P2P, SYNC, inverse, 3, taxes=taxes, batch=3) < 1e-12


def test_blocked_slab_hand_over_with_tail():
    """a one-rank and a two-rank slab plan large enough for the blocked y -> x hand-over, its Nz % CH tail included"""
    kinds = (DCT4, DST4, DCT1)
    for P in (1, 2):
        sc = describe(0, P, SL, kinds, (256, 256, 257), P, 1, P2P, SYNC, 0, 3)
        x = [s for s in sc["steps"] if s["type"] == 0 and s["label"].startswith("x")]
        assert x and x[0]["B"] < 256 * 257, "not the blocked layout"
    for inverse in (0, 1):
        assert run_type4(2, SL, kinds, (256, 256, 257), 2, 1, P2P, SYNC, inverse, 3)[0] < 1e-12
