"""Plans with untransformed (kept) axes (dfft_plan_set_transform_axes) without a GPU.

- Validation of the setter and getter, DFFT_ERR_STATE once a schedule exists, and byte-identical descriptions of plans
  whose axes are all transformed, with and without a {1, 1, 1} setter call.
- Lock-step replays of every rank's step list (step_replay.py): numpy / scipy per
  pass, a plain element copy for the copy passes (kinds 6 / 7), checked against the transform of only the transformed
  axes among the first d stages: all 8 masks for C2C and for mixed-kind R2R, the 4 R2C masks that transform z, 1-8 ranks,
  slab, Z_Then_YX and pencil, Peer2Peer and All2All, Streams (sequential), partial d, uneven splits, blocked tails,
  Bluestein lengths, batches, in-place plans and scales (each output value scaled exactly once).
- The elision rules on the step lists (DESIGN.md section 3.12), and a broken copy step that the replay rejects."""
import ctypes as C
import itertools
import json

import numpy as np
import pytest

import distributedfft_b200 as dfft
from distributedfft_b200._lib import check, lib
import step_replay as R
from step_replay import describe_raw
from test_r2r import CASES as R2R_CASES
from test_r2r_mixed import r2r_1d

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
C2C, R2C, DCT, DST, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.DST, dfft.R2HC
ERR_INVALID, ERR_STATE = -1, -4  # include/dfft.h
MASKS = list(itertools.product((0, 1), repeat=3))  # (x, y, z)
R2C_MASKS = [m for m in MASKS if m[2]]
MIXED = (R2HC, DST, DCT)


def mask_id(m):
    return "".join("t" if a else "k" for a in m)


# ---- plans ------------------------------------------------------------------------------------------------------------
def plan_of(P, decomp, transform, shape, p1, p2, axes=None, comm=P2P, send=SYNC, batch=1, inplace=False, scale=None, prec=dfft.F64, kinds=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, kinds=kinds, prec=prec, comm=comm, send=send, batch=batch, inplace=inplace,
                  axes=axes, scale=scale)


def create(rank, P, decomp, transform, shape, p1, p2, comm=P2P, send=SYNC, batch=1, inplace=False, prec=dfft.F64, kinds=None):
    """dry plan: (comm, plan); kinds: a per-axis real-to-real plan"""
    rc, msg, c, plan = R.create(plan_of(P, decomp, transform, shape, p1, p2, None, comm, send, batch, inplace, None, prec, kinds), rank)
    assert rc == 0, msg
    return c, plan


def destroy(c, plan):
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


def set_axes(plan, axes):
    return lib().dfft_plan_set_transform_axes(plan, None if axes is None else (C.c_int * 3)(*axes))


def describe(rank, P, decomp, transform, shape, p1, p2, axes, inverse, d, comm=P2P, send=SYNC, batch=1, inplace=False, scale=None,
             prec=dfft.F64, kinds=None):
    return R.describe(plan_of(P, decomp, transform, shape, p1, p2, axes, comm, send, batch, inplace, scale, prec, kinds), rank, inverse, d)


# ---- validation ---------------------------------------------------------------------------------------------------------
def test_validation_and_default():
    t = (C.c_int * 3)()
    c, plan = create(0, 1, SL, C2C, (8, 16, 32), 1, 1)
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 1, 1)
    assert lib().dfft_plan_get_transform_axes(None, t) == ERR_INVALID
    assert lib().dfft_plan_get_transform_axes(plan, None) == ERR_INVALID
    assert set_axes(None, (1, 1, 0)) == ERR_INVALID
    assert set_axes(plan, None) == ERR_INVALID
    for bad in ((2, 1, 1), (1, -1, 1), (1, 1, 3), (0, 0, 7)):
        assert set_axes(plan, bad) == ERR_INVALID, bad
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 1, 1)  # refused calls change nothing
    assert set_axes(plan, (0, 1, 1)) == 0
    assert set_axes(plan, (1, 0, 0)) == 0  # may be set again until a schedule exists
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 0, 0)
    describe_raw(plan, 0, 3)
    assert set_axes(plan, (1, 1, 1)) == ERR_STATE
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 0, 0)
    destroy(c, plan)


@pytest.mark.parametrize("inplace", [False, True])
def test_r2c_must_transform_z(inplace):
    for P, decomp, p1, p2 in ((1, SL, 1, 1), (4, PE, 2, 2)):
        c, plan = create(0, P, decomp, R2C, (8, 16, 32), p1, p2, inplace=inplace)
        for m in MASKS:
            assert set_axes(plan, m) == (0 if m[2] else ERR_INVALID), m
        destroy(c, plan)


def test_r2r_kinds_still_reported():
    c, plan = create(0, 1, SL, None, (8, 16, 32), 1, 1, kinds=MIXED)
    assert set_axes(plan, (0, 1, 1)) == 0
    k = (C.c_int * 3)()
    check(lib().dfft_plan_get_r2r_kinds(plan, k))
    assert tuple(k) == MIXED
    sc = json.loads(describe_raw(plan, 0, 3))
    assert sc["transform_axes"] == [0, 1, 1]
    destroy(c, plan)


PLANS = [  # transform, kinds
    (C2C, None), (R2C, None), (DCT, None), (None, MIXED),
]


@pytest.mark.parametrize("transform,kinds", PLANS, ids=["c2c", "r2c", "dct", "mixed"])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2)])
def test_all_transformed_descriptions_are_unchanged(P, decomp, p1, p2, transform, kinds):
    for comm, send in ((P2P, SYNC), (A2A, SYNC), (P2P, STREAMS)):
        for batch, inplace in ((1, False), (3, False), (1, True)):
            for rank in sorted({0, P - 1}):
                a = create(rank, P, decomp, transform, (16, 32, 64), p1, p2, comm, send, batch, inplace, kinds=kinds)
                b = create(rank, P, decomp, transform, (16, 32, 64), p1, p2, comm, send, batch, inplace, kinds=kinds)
                assert set_axes(b[1], (1, 1, 1)) == 0
                for inverse in (0, 1):
                    for d in (1, 2, 3):
                        da, db = describe_raw(a[1], inverse, d), describe_raw(b[1], inverse, d)
                        assert da == db, (comm, send, batch, inplace, rank, inverse, d)
                        assert "transform_axes" not in da and '"kind":6' not in da and '"kind":7' not in da
                destroy(*a)
                destroy(*b)


# ---- references ---------------------------------------------------------------------------------------------------------
def fwd_ref(x, transform, kinds, axes, d):
    """the transformed axes among the first d stages (z, y, x order), forward"""
    for axis in (2, 1, 0)[:d]:
        if not axes[axis]:
            continue
        if kinds is not None:
            x = r2r_1d(x, kinds[axis], False, axis)
        elif transform == R2C and axis == 2:
            x = np.fft.rfft(x, axis=2)
        else:
            x = np.fft.fft(x, axis=axis)
    return x


def inv_ref(X, transform, kinds, axes, d, nz):
    """the unnormalised inverse of fwd_ref (z last: C2R ends real)"""
    for axis in (0, 1, 2):
        if axis not in (2, 1, 0)[:d] or not axes[axis]:
            continue
        if kinds is not None:
            X = r2r_1d(X, kinds[axis], True, axis)
        elif transform == R2C and axis == 2:
            X = np.fft.irfft(X, n=nz, axis=2) * nz
        else:
            X = np.fft.ifft(X, axis=axis) * X.shape[axis]
    return X


def run(P, decomp, transform, shape, p1, p2, axes, inverse, d, comm=P2P, send=SYNC, kinds=None, batch=1, inplace=False, scale=None,
        prec=dfft.F64, mutate=None):
    """replays every rank's steps in lock step; returns the worst rel-L2 error of any rank's output block"""
    nx, ny, nz = shape
    p = plan_of(P, decomp, transform, shape, p1, p2, axes, comm, send, batch, inplace, scale, prec, kinds)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    assert not scheds[0]["overlapped"]
    if axes != (1, 1, 1):
        assert scheds[0]["transform_axes"] == list(axes)
    rng = np.random.default_rng(P * 1000 + nx + ny + nz + batch + 17 * axes[0] + 5 * axes[1] + axes[2] + 3 * d)
    if kinds is not None or transform == R2C:
        xg = rng.standard_normal((batch,) + shape)
    else:
        xg = rng.standard_normal((batch,) + shape) + 1j * rng.standard_normal((batch,) + shape)
    spec = np.stack([fwd_ref(xg[f], transform, kinds, axes, d) for f in range(batch)])
    want_g = np.stack([inv_ref(spec[f], transform, kinds, axes, d, nz) for f in range(batch)]) if inverse else spec
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    if prec == dfft.F32:
        s_used = float(np.float32(s_used))
    return R.error(R.replay(p, inverse, d, spec if inverse else xg, scheds, mutate), want_g * s_used)


# ---- replays --------------------------------------------------------------------------------------------------------------
GRIDS = [  # P, decomp, shape, p1, p2, comm
    (1, SL, (8, 16, 64), 1, 1, P2P),    # one rank, blocked hand-over
    (1, ZY, (8, 16, 32), 1, 1, P2P),
    (1, PE, (8, 16, 32), 1, 1, A2A),
    (3, SL, (8, 16, 64), 3, 1, A2A),    # uneven splits
    (4, ZY, (8, 4, 32), 4, 1, P2P),
    (5, SL, (16, 16, 128), 5, 1, P2P),  # uneven, blocked with a tail
    (6, PE, (8, 16, 32), 2, 3, A2A),    # z split into odd column counts
    (8, PE, (8, 16, 32), 2, 4, P2P),
    (4, PE, (8, 16, 32), 4, 1, P2P),    # P2 = 1: the z pass stays on its rank (rule 3 drops a kept z)
    (3, PE, (8, 16, 32), 3, 1, A2A),    # 8 over 3
    (4, PE, (8, 16, 32), 1, 4, A2A),    # P1 = 1
]


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_c2c_every_mask(axes, inverse):
    for P, decomp, shape, p1, p2, comm in GRIDS:
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, comm) < 1e-12, (P, decomp)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_mixed_r2r_every_mask(axes, inverse):
    for P, decomp, shape, p1, p2, comm in GRIDS:
        assert run(P, decomp, None, shape, p1, p2, axes, inverse, 3, comm, kinds=MIXED) < 1e-12, (P, decomp)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", R2C_MASKS, ids=mask_id)
def test_replay_r2c_masks(axes, inverse):
    for P, decomp, shape, p1, p2, comm in GRIDS + [(4, SL, (8, 16, 128), 4, 1, P2P), (8, PE, (16, 16, 2048), 4, 2, P2P)]:
        assert run(P, decomp, R2C, shape, p1, p2, axes, inverse, 3, comm) < 1e-12, (P, decomp)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", [(0, 1, 1), (1, 1, 0), (0, 0, 0), (1, 0, 1)], ids=mask_id)
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", R2R_CASES)
def test_replay_every_rank_count(P, decomp, shape, p1, p2, comm, send, axes, inverse):
    """1-8 ranks, every decomposition, P2P and A2A, Streams plans (sequential), odd column counts, blocked tails"""
    assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, comm, send) < 1e-12
    assert run(P, decomp, None, shape, p1, p2, axes, inverse, 3, comm, send, kinds=MIXED) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_partial(axes, inverse, d):
    """partial d: the first d stages in z, y, x order, each transformed or kept"""
    for P, decomp, shape, p1, p2, comm in ((1, SL, (8, 16, 64), 1, 1, P2P), (3, SL, (8, 16, 64), 3, 1, A2A), (6, PE, (8, 16, 32), 2, 3, P2P),
                                           (1, PE, (8, 16, 32), 1, 1, A2A)):
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, d, comm) < 1e-12
        assert run(P, decomp, None, shape, p1, p2, axes, inverse, d, comm, kinds=MIXED) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_bluestein(axes, inverse):
    for P, decomp, shape, p1, p2, comm in ((1, SL, (12, 10, 7), 1, 1, P2P), (1, SL, (6, 100, 130), 1, 1, P2P), (2, SL, (6, 100, 130), 2, 1, P2P),
                                           (1, ZY, (6, 12, 7), 1, 1, P2P), (3, ZY, (12, 10, 7), 3, 1, A2A), (6, PE, (12, 10, 7), 2, 3, P2P)):
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, comm) < 1e-12


S = (0.25, 1.0 / 3.0)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_batch_inplace_scale(axes, inverse):
    """batch 3, in-place plans and a scale that is not 1: every output value scaled exactly once"""
    for P, decomp, shape, p1, p2 in ((1, SL, (8, 16, 64), 1, 1), (1, ZY, (8, 16, 32), 1, 1), (1, PE, (8, 16, 32), 1, 1),
                                     (3, SL, (8, 16, 64), 3, 1), (4, PE, (8, 16, 32), 2, 2), (3, ZY, (8, 4, 16), 3, 1)):
        for d in (1, 3) if decomp == ZY else (1, 2, 3):  # Z_Then_YX: partial inverses are not offered
            assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, d, batch=3, scale=S) < 1e-12
            assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, d, inplace=True, scale=S) < 1e-12
            assert run(P, decomp, None, shape, p1, p2, axes, inverse, d, kinds=MIXED, inplace=True, batch=3, scale=S) < 1e-12
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, scale=S, prec=dfft.F32) < 1e-12
        if axes[2]:
            assert run(P, decomp, R2C, shape, p1, p2, axes, inverse, 3, batch=3, scale=S) < 1e-12


# ---- elision ------------------------------------------------------------------------------------------------------------
def same_view(st, inplace):
    """the same elements of the same buffer (in place, the caller's `in` and `out` are one buffer)"""
    return st["in"] == st["out"] and (st["in_user"] == st["out_user"] or (inplace and st["in_user"] > 0 and st["out_user"] > 0))


ELIDE_GRIDS = [(1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2), (3, SL, 3, 1), (4, PE, 4, 1),
               (4, PE, 1, 4)]


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("transform,kinds", [(C2C, None), (None, MIXED)], ids=["c2c", "mixed"])
def test_elision_rules(transform, kinds, inplace):
    shape = (8, 16, 64)
    for P, decomp, p1, p2 in ELIDE_GRIDS:
        for axes in MASKS:
            for inverse in (0, 1):
                for d in (1, 2, 3):
                    sc = describe(0, P, decomp, transform, shape, p1, p2, axes, inverse, d, inplace=inplace, kinds=kinds)
                    passes = [s for s in sc["steps"] if s["type"] == 0]
                    for st in passes:
                        if st["kind"] in (6, 7):
                            # rule 1: a copy that moves nothing stays only where it stores final values in place (it applies
                            # the scale)
                            assert not same_view(st, inplace) or (inplace and st["out_user"] == 2), (P, decomp, axes, inverse, d, st["label"])
                    labels = [s["label"] for s in passes]
                    # rule 3: the z pass is local on one rank, on slab ZY_Then_X and on pencil grids with P2 = 1
                    z_local = P == 1 or decomp == SL or (decomp == PE and p2 == 1)
                    if not axes[2] and d >= 2:
                        assert any(l.startswith("z ") for l in labels) != z_local, (P, decomp, p1, p2, axes, inverse, d, labels)
                    if P == 1 and not axes[0] and d == 3:  # rule 2
                        d2 = describe(0, P, decomp, transform, shape, p1, p2, axes, inverse, 2, inplace=inplace, kinds=kinds)
                        assert sc["steps"] == d2["steps"], (decomp, axes, inverse)
                        assert not any(l.startswith("x ") for l in labels)
                    if P == 1 and axes == (1, 1, 0) and d == 3:
                        assert sorted(labels) == ["x pass", "y pass"]


def test_one_rank_masks_need_few_passes():
    """one rank: each kept axis saves its pass except a kept y between two transformed axes"""
    for decomp in (SL, ZY, PE):
        for axes in MASKS:
            for inverse in (0, 1):
                sc = describe(0, 1, decomp, C2C, (8, 16, 64), 1, 1, axes, inverse, 3)
                passes = [s for s in sc["steps"] if s["type"] == 0]
                assert len(passes) <= 3 - (not axes[0]) - (not axes[2]) + (axes == (0, 0, 0)), (decomp, axes, inverse, [s["label"] for s in passes])
                assert sum(s["kind"] in (6, 7) for s in passes) <= 1


def test_streams_plans_run_sequential_schedule():
    for axes in ((0, 1, 1), (1, 0, 1), (1, 1, 0)):
        for inverse in (0, 1):
            sc = describe(0, 4, SL, C2C, (16, 8, 64), 4, 1, axes, inverse, 3, send=STREAMS)
            assert not sc["overlapped"] and all(s["stream"] == 0 for s in sc["steps"])
            sc = describe(0, 4, PE, C2C, (16, 8, 64), 2, 2, axes, inverse, 3, send=STREAMS)
            assert not sc["overlapped"]


def test_fused_and_batched_stages_need_every_axis():
    """the fused z + y stage (512^3 one-rank slab) and the batched stage (32^3) are not chosen with a kept axis"""
    for axes in ((0, 1, 1), (1, 1, 0), (1, 0, 1)):
        for inverse in (0, 1):
            sc = describe(0, 1, SL, C2C, (512, 512, 512), 1, 1, axes, inverse, 3)
            assert all(s["label"] not in ("zy pass: z phase", "yz pass: z phase") for s in sc["steps"])
            sc = describe(0, 1, SL, C2C, (32, 32, 32), 1, 1, axes, inverse, 3, batch=4)
            assert all(not s["label"].startswith("batched") for s in sc["steps"])
    full = describe(0, 1, SL, C2C, (512, 512, 512), 1, 1, None, 0, 3)
    assert any(s["label"] == "zy pass: z phase" for s in full["steps"])


def _break_copy(scheds):
    for sc in scheds:
        for st in sc["steps"]:
            if st["type"] == 0 and st["kind"] in (6, 7):
                st["out"]["segs"][0]["sA0"], st["out"]["sN"] = st["out"]["sN"], st["out"]["segs"][0]["sA0"]
                return


def test_replay_rejects_a_broken_copy():
    """negative test: a copy step with its output strides swapped does not reproduce the reference"""
    assert run(1, PE, C2C, (8, 16, 32), 1, 1, (1, 0, 1), 0, 3) < 1e-12
    try:
        err = run(1, PE, C2C, (8, 16, 32), 1, 1, (1, 0, 1), 0, 3, mutate=_break_copy)
    except (AssertionError, KeyError, IndexError):
        return
    assert err > 1e-3
