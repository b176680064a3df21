"""DCT / DST plans without a GPU.

- The R2R pass's per-line steps on the CPU (tests/emu_r2r.cpp: r2r.hpp and fft_core.cuh's stage arithmetic) against a naive
  long-double DCT / DST for every N = 2..8192, both kinds, both directions, f64 and f32, and a zero partner line.
- Length and transform validation, the work area and the domain size, and dfft_plan_describe: R2R pass kinds, real element
  sizes, the "r2r" marking, the sequential schedule also with send_method Streams.
- Lock-step replays of every rank's step list (dfft_plan_describe) with scipy's DCT / DST per pass over the reals of the
  views, checked against scipy.fft.dctn / dstn of the global array: 1-8 ranks, slab, Z_Then_YX and pencil grids, Peer2Peer
  and All2All, partial d, uneven splits with odd column counts, blocked hand-over layouts, batches, in-place plans and
  output scales (applied exactly once).  Each replay (step_replay.py) also checks the happens-before order of every
  access."""
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
from test_inplace import describe

HERE = os.path.dirname(os.path.abspath(__file__))
SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1


def test_r2r_kernel_math_matches_naive():
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "emu")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "emu_r2r.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0, r.stdout[-2000:]
        assert "fails=0" in r.stdout


def create(transform, shape, P=1, decomp=SL, p1=None, p2=1, prec=dfft.F64):
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(0, P, C.byref(c)))
    plan = C.c_void_p()
    rc = lib().dfft_plan_create(c, None, decomp, prec, transform, *shape, P if p1 is None else p1, p2, 1, C.byref(plan))
    return rc, c, plan


def destroy(c, plan):
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


@pytest.mark.parametrize("transform", [dfft.DCT, dfft.DST])
def test_length_and_transform_validation(transform):
    for shape in ((2, 2, 2), (8192, 2, 2), (2, 8192, 4), (4, 4, 8192)):
        rc, c, plan = create(transform, shape)
        assert rc == 0, shape
        destroy(c, plan)
    for shape in ((1, 4, 4), (12, 4, 4), (4, 16384, 4), (4, 4, 16384), (4, 4, 3), (96, 96, 96)):
        rc, c, plan = create(transform, shape)
        assert rc == -5, shape  # DFFT_ERR_UNSUPPORTED
        destroy(c, plan)
    rc, c, plan = create(4, (8, 8, 8))
    assert rc == -1  # not a transform
    destroy(c, plan)


@pytest.mark.parametrize("prec,es", [(dfft.F64, 8), (dfft.F32, 4)])
def test_sizes_and_layout(prec, es):
    rc, c, plan = create(dfft.DCT, (16, 32, 64), P=4, prec=prec)
    assert rc == 0
    assert lib().dfft_get_domain_size(plan) == 4 * 32 * 64 * es  # x split [4][32][64] and y split [16][8][64]
    destroy(c, plan)
    for which in range(4):  # the z extent is Nz everywhere, as for C2C
        assert dfft.layout(PE, dfft.DST, 16, 32, 64, 2, 2, 3, which) == dfft.layout(PE, dfft.C2C, 16, 32, 64, 2, 2, 3, which)


@pytest.mark.parametrize("transform,name", [(dfft.DCT, "dct"), (dfft.DST, "dst")])
@pytest.mark.parametrize("prec", [dfft.F64, dfft.F32])
def test_describe(transform, name, prec):
    for P, decomp, p1, p2 in ((1, SL, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2)):
        for send in (SYNC, STREAMS):
            for inverse in (0, 1):
                sc = describe(0, P, decomp, transform, (16, 32, 64), p1, p2, P2P, send, inverse, 3, prec=prec, inplace=False)
                assert sc["r2r"] == name and sc["esize"] == (8 if prec == dfft.F64 else 4)
                assert not sc["overlapped"] and all(s["stream"] == 0 for s in sc["steps"])
                kinds = [s["kind"] for s in sc["steps"] if s["type"] == 0]
                assert len(kinds) == 3 and set(kinds) <= {4, 5} and kinds[0 if not inverse else -1] == 4
    sc = describe(0, 1, SL, dfft.C2C, (16, 32, 64), 1, 1, P2P, SYNC, 0, 3, prec=prec, inplace=False)
    assert "r2r" not in sc


def scipy_r2r(x, transform, inverse, axis):
    f = sf.dct if transform == dfft.DCT else sf.dst
    return f(x, type=3 if inverse else 2, axis=axis)


def global_ref(x, transform, inverse, d):
    f = sf.dctn if transform == dfft.DCT else sf.dstn
    return f(x, type=3 if inverse else 2, axes={1: (2,), 2: (1, 2), 3: (0, 1, 2)}[d])


def run_r2r(P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, inplace=False, scale=None, prec=dfft.F64):
    """replays every rank's steps in lock step; returns the worst rel-L2 error of any rank's output block"""
    nx, ny, nz = shape
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=prec, comm=comm, send=send, batch=batch, inplace=inplace, scale=scale)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    assert not scheds[0]["overlapped"]
    rng = np.random.default_rng(P * 1000 + nx + ny + nz + batch)
    xg = rng.standard_normal((batch,) + shape)
    spec = np.stack([global_ref(xg[f], transform, False, d) for f in range(batch)])
    want_g = np.stack([global_ref(spec[f], transform, True, d) for f in range(batch)]) if inverse else spec
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    if prec == dfft.F32:
        s_used = float(np.float32(s_used))
    return R.error(R.replay(p, inverse, d, spec if inverse else xg, scheds), want_g * s_used)


CASES = [
    # P, decomp, shape, p1, p2, comm, send
    (1, SL, (8, 16, 64), 1, 1, P2P, SYNC),           # blocked hand-over, one rank
    (1, ZY, (8, 16, 32), 1, 1, P2P, SYNC),
    (1, PE, (8, 16, 32), 1, 1, P2P, SYNC),
    (2, SL, (8, 16, 128), 2, 1, A2A, SYNC),
    (4, SL, (16, 8, 64), 4, 1, P2P, STREAMS),        # Streams: still the sequential schedule
    (3, SL, (8, 16, 64), 3, 1, P2P, SYNC),           # uneven splits
    (3, ZY, (8, 4, 16), 3, 1, P2P, SYNC),            # z split 6 / 5 / 5: odd column counts
    (4, ZY, (8, 4, 32), 4, 1, A2A, SYNC),
    (5, SL, (16, 16, 128), 5, 1, P2P, SYNC),         # uneven, blocked with a tail
    (6, PE, (8, 16, 16), 3, 2, P2P, SYNC),
    (6, PE, (8, 16, 32), 2, 3, A2A, SYNC),           # P2 = 3: z split into odd column counts
    (8, PE, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, (16, 16, 1024), 4, 2, P2P, SYNC),        # pencil, blocked second transposition
    (7, SL, (16, 8, 32), 7, 1, A2A, SYNC),
]


@pytest.mark.parametrize("transform", [dfft.DCT, dfft.DST])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", CASES)
def test_replay_full(P, decomp, shape, p1, p2, comm, send, transform, inverse):
    assert run_r2r(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_replay_partial(d, inverse, comm):
    assert run_r2r(8, PE, dfft.DCT, (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert run_r2r(6, PE, dfft.DST, (8, 16, 16), 2, 3, comm, SYNC, inverse, d) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("transform", [dfft.DCT, dfft.DST])
def test_replay_batch_inplace_scale(transform, inverse):
    s = (0.25, 1.0 / 3.0)
    assert run_r2r(1, SL, transform, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, batch=3) < 1e-12
    assert run_r2r(3, SL, transform, (8, 16, 64), 3, 1, P2P, SYNC, inverse, 3, batch=3, scale=s) < 1e-12
    assert run_r2r(1, SL, transform, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, inplace=True, scale=s) < 1e-12
    assert run_r2r(1, PE, transform, (8, 16, 32), 1, 1, P2P, SYNC, inverse, 2, inplace=True, batch=3) < 1e-12
    assert run_r2r(4, PE, transform, (8, 16, 32), 2, 2, A2A, SYNC, inverse, 3, inplace=True, batch=3, scale=s) < 1e-12
    assert run_r2r(3, ZY, transform, (8, 4, 16), 3, 1, P2P, SYNC, inverse, 3, inplace=True, scale=s, prec=dfft.F32) < 1e-12


def test_block_width_is_tile_width_in_reals():
    """the blocked hand-over of the slab's y -> x exchange is 2 TBT reals wide, the R2R tile: one tile per block row"""
    for prec, shape in ((dfft.F64, (64, 64, 512)), (dfft.F32, (32, 32, 256)), (dfft.F64, (512, 512, 512)), (dfft.F32, (256, 256, 128))):
        sc = describe(0, 1, SL, dfft.DCT, shape, 1, 1, P2P, SYNC, 0, 3, prec=prec, inplace=False)
        x = [s for s in sc["steps"] if s["type"] == 0][-1]
        tbt = min(32, max(4 if prec == dfft.F64 else 8, 4096 // shape[0]))
        assert x["B"] == 2 * tbt, (prec, shape, x["B"])
    assert run_r2r(1, SL, dfft.DST, (32, 32, 256), 1, 1, P2P, SYNC, 0, 3, prec=dfft.F32) < 1e-12
    assert run_r2r(2, SL, dfft.DCT, (32, 32, 256), 2, 1, P2P, SYNC, 1, 3) < 1e-12
