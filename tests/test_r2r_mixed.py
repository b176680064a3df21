"""Real-to-real plans with a kind per axis (dfft_plan_create_r2r) without a GPU.

- The R2HC / HC2R pass's per-line steps on the CPU (tests/emu_r2hc.cpp: r2r.hpp and fft_core.cuh's stage arithmetic)
  against a naive long-double R2HC / HC2R for every N = 2..8192, both directions, f64 and f32, and a zero partner line.
- Kind and length validation, dfft_plan_get_r2r_kinds, and dfft_plan_describe: three DCT (DST) kinds give the DFFT_DCT
  (DFFT_DST) plan's description byte for byte; other combinations add "r2r_kinds" and a per-pass "r2r".
- Lock-step replays of every rank's step list with numpy / scipy per pass, each pass with the kind its description names,
  checked against the per-axis transform of the global array: all 27 kind combinations on a grid with three distinct
  lengths and a cubic grid with three different kinds, 1-8 ranks, slab, Z_Then_YX and pencil, Peer2Peer and All2All,
  Streams (still the sequential schedule), partial d, the odd column counts of test_r2r's cases, blocked layouts with
  tails, batches, in-place plans and output scales (applied exactly once), with the happens-before check of every access
  (step_replay.py)."""
import ctypes as C
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest
import scipy.fft as sf

import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
import step_replay as R
from step_replay import hc2r, r2hc
from test_r2r import CASES

HERE = os.path.dirname(os.path.abspath(__file__))
SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
DCT, DST, R2HC = dfft.DCT, dfft.DST, dfft.R2HC
NAMES = {DCT: "dct", DST: "dst", R2HC: "r2hc"}
ALL_KINDS = list(itertools.product((DCT, DST, R2HC), repeat=3))


def test_r2hc_kernel_math_matches_naive():
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "emu")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "emu_r2hc.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        print(r.stdout[-400:])
        assert r.returncode == 0, r.stdout[-2000:]
        assert "fails=0" in r.stdout


# ---- numpy references: the per-axis transforms (FFTW's halfcomplex format: step_replay.r2hc / hc2r) ----------------------------------------------
def r2r_1d(x, kind, inverse, axis):
    if kind == R2HC:
        return hc2r(x, axis) if inverse else r2hc(x, axis)
    f = sf.dct if kind == DCT else sf.dst
    return f(x, type=3 if inverse else 2, axis=axis)


def global_ref(x, kinds, inverse, d):
    """the first d axes in z, y, x order, each with its kind"""
    for axis in (2, 1, 0)[:d]:
        x = r2r_1d(x, kinds[axis], inverse, axis)
    return x


def test_halfcomplex_reference():
    rng = np.random.default_rng(5)
    for n in (2, 4, 8, 64):
        x = rng.standard_normal(n)
        h = r2hc(x, 0)
        X = np.fft.fft(x)
        assert np.allclose(h[:n // 2 + 1], X.real[:n // 2 + 1]) and np.allclose(h[n // 2 + 1:], X.imag[1:n // 2][::-1])
        assert np.allclose(hc2r(h, 0), n * x)


# ---- plans ------------------------------------------------------------------------------------------------------------
def create_r2r(rank, P, decomp, kinds, shape, p1, p2, comm=P2P, send=SYNC, batch=1, inplace=False, prec=dfft.F64):
    """dry plan: (rc, comm, plan)"""
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(rank, P, C.byref(c)))
    cfg = _lib.dfft_config(1, 0, comm, send, None, comm, send)
    plan = C.c_void_p()
    k = None if kinds is None else (C.c_int * 3)(*kinds)
    rc = lib().dfft_plan_create_r2r(c, C.byref(cfg), decomp, prec, k, *shape, p1, p2, batch, 1 if inplace else 0, 1, C.byref(plan))
    return rc, c, plan


def create_plain(rank, P, decomp, transform, shape, p1, p2, comm=P2P, send=SYNC, batch=1, inplace=False, prec=dfft.F64):
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(rank, P, C.byref(c)))
    cfg = _lib.dfft_config(1, 0, comm, send, None, comm, send)
    plan = C.c_void_p()
    fn = lib().dfft_plan_create_inplace if inplace else lib().dfft_plan_create_batched
    rc = fn(c, C.byref(cfg), decomp, prec, transform, *shape, p1, p2, batch, 1, C.byref(plan))
    return rc, c, plan


def destroy(c, plan):
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


def describe_raw(plan, inverse, d):
    need = C.c_size_t()
    check(lib().dfft_plan_describe(plan, inverse, d, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib().dfft_plan_describe(plan, inverse, d, buf, need.value, C.byref(need)))
    return buf.value.decode()


def describe(rank, P, decomp, kinds, shape, p1, p2, comm, send, inverse, d, batch=1, prec=dfft.F64, scale=None, inplace=False):
    p = R.Plan(P, decomp, tuple(shape), p1, p2, kinds=kinds, prec=prec, comm=comm, send=send, batch=batch, inplace=inplace, scale=scale)
    return R.describe(p, rank, inverse, d)


def test_kind_validation():
    for kinds in ((0, 2, 2), (2, 1, 2), (2, 2, 5), (4, 4, -1), (3, 7, 4)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, (8, 8, 8), 1, 1)
        assert rc == -1, kinds  # DFFT_ERR_INVALID
        destroy(c, plan)
    rc, c, plan = create_r2r(0, 1, SL, None, (8, 8, 8), 1, 1)
    assert rc == -1
    destroy(c, plan)
    for transform in (4, 5):  # a plan's kinds come only through dfft_plan_create_r2r
        for inplace in (False, True):
            rc, c, plan = create_plain(0, 1, SL, transform, (8, 8, 8), 1, 1, inplace=inplace)
            assert rc == -1, (transform, inplace)
            destroy(c, plan)
    # the single-axis call: a kind outside {DCT, DST, R2HC} is refused before anything runs
    for t in (0, 1, 5):
        assert lib().dfft_fft1d_r2r(dfft.F64, t, -1, 8, 1, 1, None, None, None) == -1


@pytest.mark.parametrize("kinds", [(R2HC, R2HC, DCT), (DST, R2HC, DCT), (R2HC, R2HC, R2HC)])
def test_length_validation(kinds):
    for shape in ((2, 2, 2), (8192, 2, 2), (2, 8192, 4), (4, 4, 8192)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, shape, 1, 1)
        assert rc == 0, shape
        destroy(c, plan)
    for shape in ((1, 4, 4), (12, 4, 4), (4, 16384, 4), (4, 4, 16384), (4, 4, 3), (96, 96, 96)):
        rc, c, plan = create_r2r(0, 1, SL, kinds, shape, 1, 1)
        assert rc == -5, shape  # DFFT_ERR_UNSUPPORTED
        destroy(c, plan)


def test_get_r2r_kinds():
    k = (C.c_int * 3)()
    for kinds in ((R2HC, R2HC, DCT), (DST, R2HC, DCT), (DCT, DCT, DCT), (R2HC, DST, DST)):
        rc, c, plan = create_r2r(0, 4, PE, kinds, (8, 16, 32), 2, 2)
        assert rc == 0
        check(lib().dfft_plan_get_r2r_kinds(plan, k))
        assert tuple(k) == kinds
        destroy(c, plan)
    for transform, want in ((DCT, 0), (DST, 0), (dfft.C2C, -1), (dfft.R2C, -1)):
        rc, c, plan = create_plain(0, 1, SL, transform, (8, 8, 8), 1, 1)
        assert rc == 0
        assert lib().dfft_plan_get_r2r_kinds(plan, k) == want
        if want == 0:
            assert tuple(k) == (transform,) * 3
        destroy(c, plan)
    assert lib().dfft_plan_get_r2r_kinds(None, k) == -1


GRIDS = [  # P, decomp, p1, p2
    (1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1),
    (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2),
    (6, SL, 6, 1), (6, ZY, 6, 1), (6, PE, 3, 2),
]


@pytest.mark.parametrize("transform", [DCT, DST])
@pytest.mark.parametrize("P,decomp,p1,p2", GRIDS)
def test_uniform_kinds_describe_as_the_dct_dst_plan(P, decomp, p1, p2, transform):
    shape = (16, 32, 64)
    for comm, send in ((P2P, SYNC), (A2A, SYNC), (P2P, STREAMS)):
        for batch, inplace in ((1, False), (3, False), (1, True)):
            for rank in sorted({0, P - 1}):
                rc, c1, a = create_r2r(rank, P, decomp, (transform,) * 3, shape, p1, p2, comm, send, batch, inplace)
                assert rc == 0
                rc, c2, b = create_plain(rank, P, decomp, transform, shape, p1, p2, comm, send, batch, inplace)
                assert rc == 0
                for inverse in (0, 1):
                    for d in (1, 2, 3):
                        da, db = describe_raw(a, inverse, d), describe_raw(b, inverse, d)
                        assert da == db, (comm, send, batch, inplace, rank, inverse, d)
                        assert "r2r_kinds" not in da
                destroy(c1, a)
                destroy(c2, b)


def test_describe_marks_kinds_per_pass():
    for kinds in ((R2HC, R2HC, DCT), (DST, R2HC, DCT), (R2HC, R2HC, R2HC), (DCT, DCT, DST)):
        for P, decomp, p1, p2 in ((1, SL, 1, 1), (4, ZY, 4, 1), (4, PE, 2, 2)):
            for send in (SYNC, STREAMS):
                for inverse in (0, 1):
                    sc = describe(0, P, decomp, kinds, (16, 32, 64), p1, p2, P2P, send, inverse, 3)
                    assert sc["r2r_kinds"] == [NAMES[k] for k in kinds]
                    assert sc["r2r"] == (NAMES[kinds[0]] if len(set(kinds)) == 1 else "mixed")
                    assert not sc["overlapped"] and all(s["stream"] == 0 for s in sc["steps"])
                    passes = [s for s in sc["steps"] if s["type"] == 0]
                    assert {s["kind"] for s in passes} <= {4, 5} and all("r2r" in s for s in passes)
                    # the z pass (CONTIG) carries the z kind: first forward, last inverse
                    z = passes[-1 if inverse else 0]
                    assert z["kind"] == 4 and z["r2r"] == NAMES[kinds[2]]


# ---- lock-step replay ---------------------------------------------------------------------------------------------------
def run_mixed(P, decomp, kinds, shape, p1, p2, comm, send, inverse, d, batch=1, inplace=False, scale=None, prec=dfft.F64):
    """replays every rank's steps in lock step, each pass with the kind its description names; returns the worst rel-L2
    error of any rank's output block against the per-axis transform of the global array"""
    nx, ny, nz = shape
    p = R.Plan(P, decomp, tuple(shape), p1, p2, kinds=kinds, prec=prec, comm=comm, send=send, batch=batch, inplace=inplace, scale=scale)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    assert not scheds[0]["overlapped"]
    rng = np.random.default_rng(P * 1000 + nx + ny + nz + batch + 7 * kinds[0] + 3 * kinds[1] + kinds[2])
    xg = rng.standard_normal((batch,) + shape)
    spec = np.stack([global_ref(xg[f], kinds, False, d) for f in range(batch)])
    want_g = np.stack([global_ref(spec[f], kinds, True, d) for f in range(batch)]) if inverse else spec
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    if prec == dfft.F32:
        s_used = float(np.float32(s_used))
    return R.error(R.replay(p, inverse, d, spec if inverse else xg, scheds), want_g * s_used)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("kinds", ALL_KINDS, ids=lambda k: "-".join(NAMES[x] for x in k))
def test_replay_every_kind_combination(kinds, inverse):
    """distinct lengths, so a pass given another axis's kind fails"""
    assert run_mixed(1, SL, kinds, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3) < 1e-12
    assert run_mixed(3, ZY, kinds, (8, 4, 16), 3, 1, A2A, SYNC, inverse, 3) < 1e-12
    assert run_mixed(4, PE, kinds, (8, 16, 32), 2, 2, P2P, SYNC, inverse, 3) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("kinds", [(DST, R2HC, DCT), (R2HC, DCT, DST), (DCT, DST, R2HC)])
def test_replay_cubic_grid_takes_kinds_from_axes(kinds, inverse):
    """one length on every axis: only the axis can tell the passes' kinds apart"""
    for P, decomp, p1, p2, comm in ((1, SL, 1, 1, P2P), (2, SL, 2, 1, A2A), (4, ZY, 4, 1, P2P), (6, PE, 3, 2, A2A)):
        assert run_mixed(P, decomp, kinds, (16, 16, 16), p1, p2, comm, SYNC, inverse, 3) < 1e-12


MIXED = [(R2HC, R2HC, DCT), (DST, R2HC, DCT), (R2HC, DST, R2HC)]


@pytest.mark.parametrize("kinds", MIXED, ids=lambda k: "-".join(NAMES[x] for x in k))
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", CASES)
def test_replay_full(P, decomp, shape, p1, p2, comm, send, inverse, kinds):
    """1-8 ranks, every decomposition, P2P and A2A, Streams, uneven splits with odd column counts, blocked tails"""
    assert run_mixed(P, decomp, kinds, shape, p1, p2, comm, send, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_replay_partial(d, inverse, comm):
    """partial d: the first d axes in z, y, x order, each with its own kind"""
    assert run_mixed(8, PE, (R2HC, R2HC, DCT), (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert run_mixed(6, PE, (DCT, DST, R2HC), (8, 16, 16), 2, 3, comm, SYNC, inverse, d) < 1e-12
    assert run_mixed(3, SL, (R2HC, DST, DCT), (8, 16, 64), 3, 1, comm, SYNC, inverse, d) < 1e-12
    assert run_mixed(1, SL, (DST, R2HC, R2HC), (8, 16, 64), 1, 1, comm, SYNC, inverse, d) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("kinds", MIXED, ids=lambda k: "-".join(NAMES[x] for x in k))
def test_replay_batch_inplace_scale(kinds, inverse):
    s = (0.25, 1.0 / 3.0)
    assert run_mixed(1, SL, kinds, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, batch=3) < 1e-12
    assert run_mixed(3, SL, kinds, (8, 16, 64), 3, 1, P2P, SYNC, inverse, 3, batch=3, scale=s) < 1e-12
    assert run_mixed(1, SL, kinds, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, inplace=True, scale=s) < 1e-12
    assert run_mixed(5, SL, kinds, (16, 16, 128), 5, 1, P2P, SYNC, inverse, 3, scale=s) < 1e-12  # blocked with a tail
    assert run_mixed(1, PE, kinds, (8, 16, 32), 1, 1, P2P, SYNC, inverse, 2, inplace=True, batch=3) < 1e-12
    assert run_mixed(4, PE, kinds, (8, 16, 32), 2, 2, A2A, SYNC, inverse, 3, inplace=True, batch=3, scale=s) < 1e-12
    assert run_mixed(3, ZY, kinds, (8, 4, 16), 3, 1, P2P, SYNC, inverse, 3, inplace=True, scale=s, prec=dfft.F32) < 1e-12
