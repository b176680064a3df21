"""Padded plans (dfft_plan_create_padded) without a GPU: validation, layouts, and a numpy replay of every rank's step list
on geometry-only plans, checked against fftn / rfftn through the index map and by the happens-before check.

A pass with "keep" transforms its N-point line and stores only the kept indices (forward), or reads only the kept indices
and zero-embeds them (inverse)."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from step_replay import describe_raw, layouts, positions

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C, DCT, DST, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.DST, dfft.R2HC
P2P, A2A = 0, 1
ERR_INVALID, ERR_UNSUPPORTED = -1, -5


def err():
    return (lib().dfft_last_error_string() or b"").decode()


def create(rank, P, decomp, transform, shape, spec, p1, p2, comm=P2P, batch=1, prec=dfft.F64):
    """dry padded plan: (rc, comm, plan); plan is None when the creator refused"""
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=prec, comm=comm, batch=batch, spectral=tuple(spec))
    rc, _, c, plan = R.create(p, rank)
    return rc, c, (plan if rc == 0 else None)


def destroy(c, plan):
    if plan is not None:
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


# ---- index map ------------------------------------------------------------------------------------------------------------
def fwd_ref(x, transform, spec, d):
    for axis in (2, 1, 0)[:d]:
        half = transform == R2C and axis == 2
        x = np.fft.rfft(x, axis=2) if half else np.fft.fft(x, axis=axis)
        x = np.take(x, positions(x.shape[axis] if not half else 2 * (x.shape[2] - 1), spec[axis], half), axis=axis)
    return x


def inv_ref(X, transform, shape, spec, d):
    for axis in (0, 1, 2):
        if axis not in (2, 1, 0)[:d]:
            continue
        half = transform == R2C and axis == 2
        n = shape[axis]
        full = list(X.shape)
        full[axis] = n // 2 + 1 if half else n
        E = np.zeros(full, dtype=np.result_type(X.dtype, np.complex128))  # long double stays long double
        idx = [slice(None)] * 3
        idx[axis] = positions(n, spec[axis], half)
        E[tuple(idx)] = X
        X = np.fft.irfft(E, n=n, axis=2) * n if half else np.fft.ifft(E, axis=axis) * n
    return X


# ---- replay ---------------------------------------------------------------------------------------------------------------
def replay(P, decomp, transform, shape, spec, p1, p2, inverse, d, comm=P2P, batch=1, scale=None, mutate=None):
    """replays every rank's steps in lock step; returns the worst rel-L2 error of any rank's output block"""
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, comm=comm, batch=batch, spectral=tuple(spec), scale=scale)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    padded = tuple(spec) != tuple(shape)
    assert not scheds[0]["overlapped"]
    assert ("spectral" in scheds[0]) == padded and (not padded or scheds[0]["spectral"] == list(spec))
    rng = np.random.default_rng(sum(shape) + 7 * sum(spec) + P + 3 * d + inverse)
    if transform == R2C:
        xg = rng.standard_normal((batch,) + shape)
    else:
        xg = rng.standard_normal((batch,) + shape) + 1j * rng.standard_normal((batch,) + shape)
    spec_g = np.stack([fwd_ref(xg[f], transform, spec, d) for f in range(batch)])
    want_g = np.stack([inv_ref(spec_g[f], transform, shape, spec, d) for f in range(batch)]) if inverse else spec_g
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    return R.error(R.replay(p, inverse, d, spec_g if inverse else xg, scheds, mutate), want_g * s_used)


# ---- validation -----------------------------------------------------------------------------------------------------------
def test_validation():
    def rc(decomp=SL, transform=C2C, shape=(8, 16, 32), spec=(5, 11, 21), P=1, p1=1, p2=1):
        r, c, plan = create(0, P, decomp, transform, shape, spec, p1, p2)
        destroy(c, plan)
        return r
    assert rc() == 0
    assert rc(transform=R2C) == 0
    assert rc(transform=DCT) == ERR_UNSUPPORTED
    assert rc(transform=DST) == ERR_UNSUPPORTED
    assert rc(transform=R2HC) == ERR_INVALID
    for bad in ((0, 16, 32), (8, 0, 32), (8, 16, 0), (9, 16, 32), (8, 17, 32), (8, 16, 33)):
        assert rc(spec=bad) == ERR_INVALID, bad
    # Bluestein axes keep K = N
    assert rc(shape=(8, 12, 32), spec=(5, 12, 21)) == 0
    assert rc(shape=(8, 12, 32), spec=(5, 11, 21)) == ERR_UNSUPPORTED
    # a spectral split that leaves a rank without data
    assert rc(decomp=SL, P=4, p1=4, spec=(8, 3, 32)) == ERR_INVALID and "without data" in err()
    assert rc(decomp=ZY, P=4, p1=4, spec=(8, 16, 3)) == ERR_INVALID and "without data" in err()
    assert rc(decomp=PE, P=4, p1=2, p2=2, transform=R2C, spec=(8, 16, 1)) == ERR_INVALID and "without data" in err()
    assert rc(decomp=PE, P=4, p1=2, p2=2, transform=R2C, spec=(8, 16, 2)) == 0
    # transform axes: only {1,1,1} once some K < N
    r, c, plan = create(0, 1, SL, C2C, (8, 16, 32), (5, 16, 32), 1, 1)
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(1, 1, 1)) == 0
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == ERR_UNSUPPORTED
    k = (C.c_size_t * 3)()
    check(lib().dfft_plan_get_spectral_size(plan, k))
    assert tuple(k) == (5, 16, 32)
    destroy(c, plan)
    r, c, plan = create(0, 1, SL, C2C, (8, 16, 32), (8, 16, 32), 1, 1)
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == 0
    destroy(c, plan)


def test_tune_has_one_candidate_and_fused_stages_are_off():
    # a one-rank 512^3 C2C slab plan selects the fused z + y stage; its padded twin does not
    r, c, plan = create(0, 1, SL, C2C, (512, 512, 512), (341, 341, 341), 1, 1)
    assert r == 0
    for inverse in (0, 1):
        sc = json.loads(describe_raw(plan, inverse, 3))
        labels = [s["label"].replace(" (tail)", "") for s in sc["steps"] if s["type"] == 0]
        assert sorted(set(labels)) == ["x pass", "y pass", "z pass"], labels
        assert all(s.get("keep") == 341 for s in sc["steps"] if s["type"] == 0)
    destroy(c, plan)
    r, c, plan = create(0, 1, SL, C2C, (32, 32, 32), (21, 21, 21), 1, 1, batch=4)
    assert r == 0
    assert "batched pass" not in describe_raw(plan, 0, 3)
    destroy(c, plan)


@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2),
                                            (3, PE, 3, 1)])
def test_identity_descriptions(P, decomp, p1, p2, transform):
    shape = (16, 32, 64)
    for comm in (P2P, A2A):
        for batch in (1, 3):
            for rank in sorted({0, P - 1}):
                c = C.c_void_p()
                check(lib().dfft_comm_create_dry(rank, P, C.byref(c)))
                cfg = _lib.dfft_config(1, 0, comm, 0, None, comm, 0)
                a = C.c_void_p()
                check(lib().dfft_plan_create_batched(c, C.byref(cfg), decomp, dfft.F64, transform, *shape, p1, p2, batch, 1, C.byref(a)))
                r, c2, b = create(rank, P, decomp, transform, shape, shape, p1, p2, comm, batch)
                assert r == 0
                for inverse in (0, 1):
                    for d in (1, 2, 3):
                        assert describe_raw(a, inverse, d) == describe_raw(b, inverse, d), (comm, batch, rank, inverse, d)
                assert lib().dfft_get_work_size_device(a) == lib().dfft_get_work_size_device(b)
                lib().dfft_plan_destroy(a)
                destroy(c, None)
                destroy(c2, b)


# ---- layouts --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("decomp", [SL, ZY, PE])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 6, 8])
def test_layouts_tile_the_domains(P, decomp, transform):
    shape, spec = (16, 32, 64), (11, 21, 43)
    grids = [(P, 1)] if decomp != PE else [(a, P // a) for a in range(1, P + 1) if P % a == 0]
    kzc = spec[2] // 2 + 1 if transform == R2C else spec[2]
    nzc = shape[2] // 2 + 1 if transform == R2C else shape[2]
    for p1, p2 in grids:
        lays = []
        for r in range(P):
            rc, c, plan = create(r, P, decomp, transform, shape, spec, p1, p2)
            assert rc == 0, err()
            lays.append(layouts(plan))
            work = lib().dfft_get_work_size_device(plan)
            destroy(c, plan)
            rc, c, plan = create(r, P, decomp, transform, shape, shape, p1, p2)
            assert work <= lib().dfft_get_work_size_device(plan)
            destroy(c, plan)
        for w in range(4):
            ext = [(shape[0], shape[1], shape[2]), (shape[0], shape[1], kzc), (shape[0], spec[1], kzc), (spec[0], spec[1], kzc)][w]
            cover = np.zeros(ext, dtype=np.int64)
            for r in range(P):
                (s, o) = lays[r][w]
                cover[o[0]:o[0] + s[0], o[1]:o[1] + s[1], o[2]:o[2] + s[2]] += 1
            assert (cover == 1).all(), (p1, p2, w)
        assert nzc >= kzc


# ---- replays --------------------------------------------------------------------------------------------------------------
GRIDS = [  # P, decomp, p1, p2
    (1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1),
    (2, SL, 2, 1), (3, SL, 3, 1), (4, SL, 4, 1), (8, SL, 8, 1),
    (2, ZY, 2, 1), (4, ZY, 4, 1), (5, ZY, 5, 1),
    (4, PE, 2, 2), (6, PE, 3, 2), (8, PE, 4, 2), (4, PE, 1, 4),
]
SPECS = [  # shape, spec: odd and even K, K = 1, K = N on some axes
    ((16, 32, 64), (11, 21, 43)),
    ((16, 32, 64), (10, 32, 42)),
    ((16, 16, 64), (16, 9, 64)),
    ((8, 16, 32), (1, 16, 21)),
]


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("P,decomp,p1,p2", GRIDS)
def test_replay(P, decomp, p1, p2, transform, comm, inverse):
    for shape, spec in SPECS:
        if transform == R2C and P > 1 and decomp != SL and (spec[2] // 2 + 1) < (P if decomp == ZY else p2):
            continue
        if P > 1 and spec[1] < (P if decomp == SL else p1):
            continue
        assert replay(P, decomp, transform, shape, spec, p1, p2, inverse, 3, comm) < 1e-12, (shape, spec)


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2), (6, PE, 3, 2)])
def test_replay_partial(P, decomp, p1, p2, inverse, d):
    if decomp == ZY and inverse and d == 2:
        pytest.skip("the Z_Then_YX inverse runs its y, x and z passes for d = 2 as for d = 3 (ordinary plans alike)")
    for transform in (C2C, R2C):
        for comm in (P2P, A2A):
            assert replay(P, decomp, transform, (16, 32, 64), (11, 21, 43), p1, p2, inverse, d, comm) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (3, SL, 3, 1), (3, ZY, 3, 1), (6, PE, 3, 2)])
def test_replay_batch_scale_uneven_tails(P, decomp, p1, p2, inverse):
    # uneven spectral splits and blocked tails: 43 z columns over 2 or 3 ranks, 21 y rows over 3
    for transform in (C2C, R2C):
        assert replay(P, decomp, transform, (16, 32, 128), (11, 21, 85), p1, p2, inverse, 3, P2P, batch=3, scale=(0.25, 1.0 / 3.0)) < 1e-12


def drop_rendezvous(scheds):
    """schedule mutation: remove every rendezvous but the entry one"""
    for sc in scheds:
        sc["steps"] = [st for st in sc["steps"] if st["type"] != 1 or st["group"] == 0]


@pytest.mark.parametrize("inverse", [0, 1])
def test_slot_rule_catches_a_missing_rendezvous(inverse):
    """the replay's slot rule holds padded plans too: without the rendezvous of its transpositions, a pass reads a slot that
    a peer stored into"""
    case = (4, SL, C2C, (16, 32, 64), (11, 21, 43), 4, 1, inverse, 3)
    assert replay(*case) < 1e-12
    with pytest.raises(AssertionError, match="without a rendezvous"):
        replay(*case, mutate=drop_rendezvous)
