"""Pruned plans (dfft_plan_create_pruned) without a GPU: validation, layouts, the identity with padded and ordinary plans, and
a numpy replay of every rank's step list on geometry-only plans, checked against fftn / rfftn of the zero-embedded field
and by the happens-before check.

A pass with "data" reads only the first `data` points of its physical side and takes the rest as zero (forward), or
transforms its N-point line and stores only the first `data` points (inverse)."""
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


def plan_of(P, decomp, transform, shape, data, spec, p1, p2, comm=P2P, batch=1, scale=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, comm=comm, batch=batch, scale=scale,
                 data=tuple(data), spectral=None if spec is None else tuple(spec))


def create(rank, P, decomp, transform, shape, data, spec, p1, p2, comm=P2P, batch=1):
    """dry pruned plan: (rc, comm, plan); plan is None when the creator refused"""
    rc, _, c, plan = R.create(plan_of(P, decomp, transform, shape, data, spec, p1, p2, comm, batch), rank)
    return rc, c, (plan if rc == 0 else None)


def destroy(c, plan):
    if plan is not None:
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


# ---- index map ------------------------------------------------------------------------------------------------------------
def fwd_ref(x, transform, shape, spec, d):
    """the first d axes (z, y, x order) of the m-block x zero-embedded to N, transformed and truncated to K"""
    for axis in (2, 1, 0)[:d]:
        half = transform == R2C and axis == 2
        pad = [(0, 0)] * 3
        pad[axis] = (0, shape[axis] - x.shape[axis])
        x = np.pad(x, pad)
        x = np.fft.rfft(x, axis=2) if half else np.fft.fft(x, axis=axis)
        x = np.take(x, positions(shape[axis], spec[axis], half), axis=axis)
    return x


def inv_ref(X, transform, shape, data, spec, d):
    """the unnormalised inverse of the zero-embedded spectrum along the first d axes, truncated to the data block"""
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
        X = np.take(X, np.arange(data[axis]), axis=axis)
    return X


# ---- replay ---------------------------------------------------------------------------------------------------------------
def replay(P, decomp, transform, shape, data, spec, p1, p2, inverse, d, comm=P2P, batch=1, scale=None):
    """replays every rank's steps in lock step; returns the worst rel-L2 error of any rank's output block"""
    spec = tuple(shape) if spec is None else tuple(spec)
    p = plan_of(P, decomp, transform, shape, data, spec, p1, p2, comm, batch, scale)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    pruned = tuple(data) != tuple(shape)
    assert not scheds[0]["overlapped"]
    assert ("data" in scheds[0]) == pruned and (not pruned or scheds[0]["data"] == list(data))
    rng = np.random.default_rng(sum(shape) + 7 * sum(data) + 3 * sum(spec) + P + 3 * d + inverse)
    if transform == R2C:
        xg = rng.standard_normal((batch,) + tuple(data))
    else:
        xg = rng.standard_normal((batch,) + tuple(data)) + 1j * rng.standard_normal((batch,) + tuple(data))
    spec_g = np.stack([fwd_ref(xg[f], transform, shape, spec, d) for f in range(batch)])
    want_g = np.stack([inv_ref(spec_g[f], transform, shape, data, spec, d) for f in range(batch)]) if inverse else spec_g
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    return R.error(R.replay(p, inverse, d, spec_g if inverse else xg, scheds), want_g * s_used)


# ---- validation -----------------------------------------------------------------------------------------------------------
def test_validation():
    def rc(decomp=SL, transform=C2C, shape=(8, 16, 32), data=(5, 11, 20), spec=None, P=1, p1=1, p2=1):
        r, c, plan = create(0, P, decomp, transform, shape, data, spec, p1, p2)
        destroy(c, plan)
        return r
    assert rc() == 0
    assert rc(transform=R2C) == 0
    assert rc(spec=(3, 16, 21)) == 0
    assert rc(transform=DCT) == ERR_UNSUPPORTED and "pruned plans are C2C or R2C" in err()
    assert rc(transform=DST) == ERR_UNSUPPORTED
    assert rc(transform=R2HC) == ERR_INVALID
    for bad in ((0, 16, 32), (8, 0, 32), (8, 16, 0), (9, 16, 32), (8, 17, 32), (8, 16, 33)):
        assert rc(data=bad) == ERR_INVALID and "data size" in err(), bad
    # the spectral arguments of padded plans are checked as there
    assert rc(spec=(8, 16, 33)) == ERR_INVALID and "spectral size" in err()
    # Bluestein axes keep M = N
    assert rc(shape=(8, 12, 32), data=(5, 12, 20)) == 0
    assert rc(shape=(8, 12, 32), data=(5, 11, 20)) == ERR_UNSUPPORTED and "not a power of two" in err()
    # real rows move as pairs
    assert rc(transform=R2C, data=(5, 11, 21)) == ERR_UNSUPPORTED and "even" in err()
    assert rc(transform=C2C, data=(5, 11, 21)) == 0
    # a data split that leaves a rank without data
    assert rc(decomp=SL, P=4, p1=4, data=(3, 16, 32)) == ERR_INVALID and "without data" in err()
    assert rc(decomp=ZY, P=4, p1=4, data=(3, 16, 32)) == ERR_INVALID and "without data" in err()
    assert rc(decomp=PE, P=4, p1=1, p2=4, data=(8, 3, 32)) == ERR_INVALID and "without data" in err()
    assert rc(decomp=PE, P=4, p1=1, p2=4, data=(8, 4, 32)) == 0
    # no in-place, boxed or interleaved form: the creator has no such argument.  Transform axes and strides:
    r, c, plan = create(0, 1, SL, C2C, (8, 16, 32), (5, 16, 32), None, 1, 1)
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(1, 1, 1)) == 0
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == ERR_UNSUPPORTED and "pruned" in err()
    assert lib().dfft_plan_set_strides(plan, (C.c_longlong * 3)(10 * 16 * 32, 16 * 32, 32), None) == ERR_UNSUPPORTED and "pruned" in err()
    m, k = (C.c_size_t * 3)(), (C.c_size_t * 3)()
    check(lib().dfft_plan_get_data_size(plan, m))
    check(lib().dfft_plan_get_spectral_size(plan, k))
    assert tuple(m) == (5, 16, 32) and tuple(k) == (8, 16, 32)
    destroy(c, plan)
    # m = N: transform axes and strides as for any plan
    r, c, plan = create(0, 1, SL, C2C, (8, 16, 32), (8, 16, 32), (5, 16, 32), 1, 1)
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(1, 1, 1)) == 0
    check(lib().dfft_plan_get_data_size(plan, m))
    assert tuple(m) == (8, 16, 32)
    destroy(c, plan)
    # every other plan reports its grid
    c, a = C.c_void_p(), C.c_void_p()
    check(lib().dfft_comm_create_dry(0, 1, C.byref(c)))
    check(lib().dfft_plan_create(c, None, SL, dfft.F64, C2C, 8, 16, 32, 1, 1, 1, C.byref(a)))
    check(lib().dfft_plan_get_data_size(a, m))
    assert tuple(m) == (8, 16, 32)
    lib().dfft_plan_destroy(a)
    destroy(c, None)


def test_sequential_schedule_only():
    # a one-rank 512^3 C2C slab plan selects the fused z + y stage; its pruned twin does not
    r, c, plan = create(0, 1, SL, C2C, (512, 512, 512), (256, 256, 256), None, 1, 1)
    assert r == 0
    for inverse in (0, 1):
        sc = json.loads(describe_raw(plan, inverse, 3))
        assert sc["data"] == [256, 256, 256] and "spectral" not in sc
        labels = [s["label"].replace(" (tail)", "") for s in sc["steps"] if s["type"] == 0]
        assert sorted(set(labels)) == ["x pass", "y pass", "z pass"], labels
        assert all(s.get("data") == 256 and "keep" not in s for s in sc["steps"] if s["type"] == 0)
    destroy(c, plan)
    r, c, plan = create(0, 1, SL, C2C, (32, 32, 32), (16, 16, 16), None, 1, 1, batch=4)
    assert r == 0
    assert "batched pass" not in describe_raw(plan, 0, 3)
    destroy(c, plan)
    # one axis with m < N is enough to leave the fused stage, and only that axis's pass carries "data"
    r, c, plan = create(0, 1, SL, C2C, (512, 512, 512), (512, 512, 200), None, 1, 1)
    sc = json.loads(describe_raw(plan, 0, 3))
    assert [s.get("data") for s in sc["steps"] if s["type"] == 0 and s["label"] != "x pass (tail)"][:1] == [200]
    assert all("data" not in s for s in sc["steps"] if s["type"] == 0 and s["label"].startswith(("y pass", "x pass")))
    destroy(c, plan)


# ---- identity -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2),
                                            (3, PE, 3, 1)])
def test_identity_descriptions(P, decomp, p1, p2, transform):
    """data = N (or NULL) makes the padded plan of the same spectral, and the ordinary plan when both are full"""
    shape, spec = (16, 32, 64), (11, 21, 43)
    for comm in (P2P, A2A):
        for batch in (1, 3):
            for rank in sorted({0, P - 1}):
                c = C.c_void_p()
                check(lib().dfft_comm_create_dry(rank, P, C.byref(c)))
                cfg = _lib.dfft_config(1, 0, comm, 0, None, comm, 0)
                a, b = C.c_void_p(), C.c_void_p()
                check(lib().dfft_plan_create_batched(c, C.byref(cfg), decomp, dfft.F64, transform, *shape, p1, p2, batch, 1, C.byref(a)))
                check(lib().dfft_plan_create_padded(c, C.byref(cfg), decomp, dfft.F64, transform, *shape, *spec, p1, p2, batch, 1, C.byref(b)))
                N = (C.c_size_t * 3)(*shape)
                pairs = []
                for ref, data, k in ((a, N, None), (a, None, None), (a, N, N), (b, N, (C.c_size_t * 3)(*spec)), (b, None, (C.c_size_t * 3)(*spec))):
                    q = C.c_void_p()
                    check(lib().dfft_plan_create_pruned(c, C.byref(cfg), decomp, dfft.F64, transform, *shape, data, k, p1, p2, batch, 1, C.byref(q)))
                    pairs.append((ref, q))
                for ref, q in pairs:
                    for inverse in (0, 1):
                        for d in (1, 2, 3):
                            assert describe_raw(ref, inverse, d) == describe_raw(q, inverse, d), (comm, batch, rank, inverse, d)
                    assert lib().dfft_get_work_size_device(ref) == lib().dfft_get_work_size_device(q)
                    assert lib().dfft_get_domain_size(ref) == lib().dfft_get_domain_size(q)
                    lib().dfft_plan_destroy(q)
                lib().dfft_plan_destroy(a)
                lib().dfft_plan_destroy(b)
                destroy(c, None)


# ---- layouts --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("decomp", [SL, ZY, PE])
@pytest.mark.parametrize("P", [1, 2, 3, 4, 6, 8])
def test_layouts_tile_the_domains(P, decomp, transform):
    """m on the axes not yet transformed, K on the transformed ones; the work area never exceeds the N plan's"""
    shape, data, spec = (16, 32, 64), (9, 17, 34), (11, 21, 43)
    grids = [(P, 1)] if decomp != PE else [(a, P // a) for a in range(1, P + 1) if P % a == 0]
    kzc = spec[2] // 2 + 1 if transform == R2C else spec[2]
    for p1, p2 in grids:
        lays = []
        for r in range(P):
            rc, c, plan = create(r, P, decomp, transform, shape, data, spec, p1, p2)
            assert rc == 0, err()
            lays.append(layouts(plan))
            work = lib().dfft_get_work_size_device(plan)
            destroy(c, plan)
            rc, c, plan = create(r, P, decomp, transform, shape, shape, spec, p1, p2)
            assert work <= lib().dfft_get_work_size_device(plan)
            destroy(c, plan)
        for w in range(4):
            ext = [data, (data[0], data[1], kzc), (data[0], spec[1], kzc), (spec[0], spec[1], kzc)][w]
            cover = np.zeros(ext, dtype=np.int64)
            for r in range(P):
                (s, o) = lays[r][w]
                cover[o[0]:o[0] + s[0], o[1]:o[1] + s[1], o[2]:o[2] + s[2]] += 1
            assert (cover == 1).all(), (p1, p2, w)


def test_physical_buffers_and_work_area_shrink():
    """the caller's physical buffer of a one-rank 512^3 plan with 256^3 data is 8x smaller; the work area is the larger of
    the intermediates and the output"""
    shape, data = (512, 512, 512), (256, 256, 256)
    for transform in (C2C, R2C):
        rc, c, plan = create(0, 1, SL, transform, shape, data, None, 1, 1)
        assert rc == 0
        (s_in, _), _, (s2, _), (s3, _) = layouts(plan)
        assert s_in == list(data) and s2 == [256, 512, shape[2] // 2 + 1 if transform == R2C else 512]
        assert s3 == [512, 512, shape[2] // 2 + 1 if transform == R2C else 512]
        pruned_work = lib().dfft_get_work_size_device(plan)
        destroy(c, plan)
        rc, c, plan = create(0, 1, SL, transform, shape, shape, None, 1, 1)
        assert pruned_work <= lib().dfft_get_work_size_device(plan)
        destroy(c, plan)


# ---- transposition volume -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("P", [2, 4])
def test_slab_forward_transposition_moves_the_data_planes_only(P, transform):
    """the slab forward all-to-all carries mx * Ky * Kzc elements (the x planes beyond mx are zero and stay home)"""
    shape, data, spec = (32, 32, 64), (16, 16, 32), (32, 21, 43)
    kzc = spec[2] // 2 + 1 if transform == R2C else spec[2]
    for dat, want in ((data, data[0] * spec[1] * kzc), (shape, shape[0] * spec[1] * kzc)):
        p = plan_of(P, SL, transform, shape, dat, spec, P, 1, A2A)
        total = 0
        for r in range(P):
            sc = R.describe(p, r, 0, 3)
            a2a = [st for st in sc["steps"] if st["type"] == 2]
            assert len(a2a) == 1
            total += sum(peer["scount"] for peer in a2a[0]["peers"])
        assert total == want, (dat, total, want)


# ---- replays --------------------------------------------------------------------------------------------------------------
GRIDS = [  # P, decomp, p1, p2
    (1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1),
    (2, SL, 2, 1), (3, SL, 3, 1), (4, SL, 4, 1), (8, SL, 8, 1),
    (2, ZY, 2, 1), (4, ZY, 4, 1), (5, ZY, 5, 1),
    (4, PE, 2, 2), (6, PE, 3, 2), (8, PE, 4, 2), (4, PE, 1, 4),
]
CASES = [  # shape, data, spectral: odd and even m, m = 1, m = N on some axes, m < N together with K < N
    ((16, 32, 64), (8, 16, 32), None),
    ((16, 32, 64), (9, 17, 34), None),
    ((16, 16, 64), (16, 9, 64), None),
    ((8, 16, 32), (8, 16, 2), None),
    ((16, 32, 64), (9, 11, 30), (11, 21, 43)),
    ((16, 16, 64), (8, 16, 20), (16, 9, 33)),
]


def fits(P, decomp, p1, p2, transform, shape, data, spec):
    """every rank holds data on every split axis"""
    spec = shape if spec is None else spec
    kzc = spec[2] // 2 + 1 if transform == R2C else spec[2]
    if P > 1 and decomp != SL and kzc < (P if decomp == ZY else p2):
        return False
    if P > 1 and spec[1] < (P if decomp == SL else p1):
        return False
    return data[0] >= p1 and (decomp != PE or data[1] >= p2)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("P,decomp,p1,p2", GRIDS)
def test_replay(P, decomp, p1, p2, transform, comm, inverse):
    for shape, data, spec in CASES:
        if not fits(P, decomp, p1, p2, transform, shape, data, spec):
            continue
        assert replay(P, decomp, transform, shape, data, spec, p1, p2, inverse, 3, comm) < 1e-12, (shape, data, spec)


def test_replay_m_equal_one():
    for transform in (C2C, R2C):
        for inverse in (0, 1):
            for decomp in (SL, ZY, PE):
                assert replay(1, decomp, transform, (8, 16, 32), (1, 1, 2), None, 1, 1, inverse, 3) < 1e-12
                assert replay(1, decomp, C2C, (8, 16, 32), (1, 1, 1), (3, 5, 7), 1, 1, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2), (6, PE, 3, 2)])
def test_replay_partial(P, decomp, p1, p2, inverse, d):
    if decomp == ZY and inverse and d == 2:
        pytest.skip("the Z_Then_YX inverse runs its y, x and z passes for d = 2 as for d = 3 (ordinary plans alike)")
    for transform in (C2C, R2C):
        for comm in (P2P, A2A):
            for spec in (None, (11, 21, 43)):
                assert replay(P, decomp, transform, (16, 32, 64), (9, 17, 30), spec, p1, p2, inverse, d, comm) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (3, SL, 3, 1), (3, ZY, 3, 1), (6, PE, 3, 2)])
def test_replay_batch_scale_uneven_tails(P, decomp, p1, p2, inverse):
    # uneven data splits (11 x planes over 3 ranks, 13 y rows over 2) and blocked tails (43 z columns over 2 or 3 ranks)
    for transform in (C2C, R2C):
        for spec in (None, (11, 21, 85)):
            assert replay(P, decomp, transform, (16, 32, 128), (11, 13, 64), spec, p1, p2, inverse, 3, P2P, batch=3,
                          scale=(0.25, 1.0 / 3.0)) < 1e-12
