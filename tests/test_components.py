"""Interleaved multi-component plans (dfft_plan_create_interleaved) without a GPU: argument checks, the C = 1 identity,
sizes, and CPU replays of every rank's step list.

The replay runs the step lists dfft_plan_describe returns for every rank through step_replay.py, on [X][Y][Z][C] inputs
with a distinct input per field.  The interleaved z pass (kind 8) has the TILED view mapping with b the component.  Every field's block of every
component must match the oracle, and every step may only touch the caller's memory of its own field."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import check, lib
from oracle import dft_oracle as O

from test_batch import describe_batched
from test_padded import drop_rendezvous
from test_schedule_emulation import A2A, P2P, PE, SL, SYNC, ZY

HERE = os.path.dirname(os.path.abspath(__file__))
SIZE_MAX = (1 << 64) - 1
ILV = 8  # PASS_C2C_ILV


def plan_of(P, decomp, transform, shape, p1, p2, comps, batch=1, comm_method=P2P, prec=None, scale=1.0):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=dfft.F64 if prec is None else prec, comm=comm_method, batch=batch,
                  components=comps, scale=None if scale == 1.0 else (scale, scale))


def create(rank, P, decomp, transform, shape, p1, p2, comps, batch=1, comm_method=P2P, prec=None):
    """dry interleaved plan: (rc, message, comm, plan)"""
    return R.create(plan_of(P, decomp, transform, shape, p1, p2, comps, batch, comm_method, prec), rank)


def describe_ilv(rank, P, decomp, transform, shape, p1, p2, comps, batch, comm_method, inverse, d, scale=1.0, prec=None):
    return R.describe(plan_of(P, decomp, transform, shape, p1, p2, comps, batch, comm_method, prec, scale), rank, inverse, d)


def run_interleaved(P, decomp, shape, p1, p2, comm_method, inverse, d, comps, batch=1, scale=1.0, transform=dfft.C2C, mutate=None):
    """Replays an interleaved exec on every rank; returns the worst rel-L2 error over fields, components and ranks.  R2C /
    C2R: the z pass is the interleaved R2C / C2R pass (kinds 9 / 10) whose real side is counted in reals."""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    p = plan_of(P, decomp, transform, shape, p1, p2, comps, batch, comm_method, scale=scale)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    assert all(s.get("components", 1) == comps for s in scheds)
    xs, specs = [], []
    for f in range(batch):
        if c2c:
            x = O.complex_input((nx, ny, nz * comps), seed=99 + f).reshape(nx, ny, nz, comps)
        else:
            x = O.real_input((nx, ny, nz * comps), seed=99 + f).reshape(nx, ny, nz, comps)
        xs.append(x)
        ft = O.fft_c2c if c2c else O.fft_r2c
        specs.append(np.stack([ft(np.ascontiguousarray(x[..., c]), d) for c in range(comps)], axis=-1))
    n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
    x, want = (specs, [x * n * scale for x in xs]) if inverse else (xs, [s * scale for s in specs])
    return R.error(R.replay(p, inverse, d, x, scheds, mutate), want)


CASES = [
    # P, decomp, shape, p1, p2, comm, C
    (1, SL, (8, 16, 64), 1, 1, P2P, 3),       # blocked hand-over, one rank
    (1, ZY, (8, 8, 32), 1, 1, P2P, 2),
    (1, PE, (8, 8, 16), 1, 1, P2P, 17),       # C above the tile width: the TILED kernel's mapping, same view
    (2, SL, (8, 8, 128), 2, 1, P2P, 5),
    (3, SL, (9, 12, 64), 3, 1, P2P, 4),       # uneven splits, blocked with tails
    (4, SL, (16, 8, 64), 4, 1, A2A, 3),
    (4, ZY, (8, 4, 16), 4, 1, P2P, 8),
    (3, ZY, (6, 4, 16), 3, 1, A2A, 5),        # uneven z split
    (8, PE, (16, 8, 16), 4, 2, A2A, 2),
    (6, PE, (12, 9, 64), 3, 2, P2P, 3),       # uneven pencil, blocked with tails
    (4, PE, (8, 8, 128), 2, 2, P2P, 17),
    (2, SL, (12, 10, 32), 2, 1, P2P, 3),      # Bluestein x and y
    (4, PE, (12, 6, 32), 2, 2, A2A, 5),       # Bluestein x and y on a pencil
]


@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,comps", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_interleaved_schedules(P, decomp, shape, p1, p2, comm, comps, inverse):
    assert run_interleaved(P, decomp, shape, p1, p2, comm, inverse, 3, comps) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_interleaved_partial_schedules(d, inverse, comm):
    assert run_interleaved(8, PE, (8, 16, 32), 2, 4, comm, inverse, d, 3) < 1e-12
    # Z_Then_YX: the forward only (its d = 2 inverse runs all three stages, as for every plan)
    if not inverse or d == 1:
        assert run_interleaved(4, ZY, (8, 8, 16), 4, 1, comm, inverse, d, 5) < 1e-12
    assert run_interleaved(2, SL, (8, 8, 64), 2, 1, comm, inverse, d, 2) < 1e-12


R2C_CASES = [
    # P, decomp, shape, p1, p2, comm, C — odd and even C, multi-segment z scatter / gather, blocked tails
    (1, SL, (8, 16, 64), 1, 1, P2P, 3),
    (1, PE, (8, 8, 16), 1, 1, P2P, 2),
    (2, SL, (8, 8, 128), 2, 1, P2P, 5),
    (3, SL, (8, 16, 64), 3, 1, A2A, 4),
    (4, ZY, (8, 4, 32), 4, 1, P2P, 7),
    (3, ZY, (8, 4, 16), 3, 1, A2A, 6),
    (8, PE, (16, 8, 16), 4, 2, A2A, 2),
    (6, PE, (16, 8, 64), 3, 2, P2P, 3),
    (4, PE, (8, 8, 128), 2, 2, P2P, 17),
]


@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,comps", R2C_CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_interleaved_r2c_schedules(P, decomp, shape, p1, p2, comm, comps, inverse):
    """the interleaved R2C / C2R z pass and the complex passes behind it"""
    assert run_interleaved(P, decomp, shape, p1, p2, comm, inverse, 3, comps, transform=dfft.R2C) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
def test_interleaved_r2c_partial_batch_scale(d, inverse):
    assert run_interleaved(8, PE, (8, 16, 32), 2, 4, P2P, inverse, d, 3, transform=dfft.R2C) < 1e-12
    assert run_interleaved(2, SL, (8, 8, 64), 2, 1, A2A, inverse, d, 2, batch=2, scale=0.375, transform=dfft.R2C) < 1e-12
    assert run_interleaved(4, SL, (8, 8, 32), 4, 1, P2P, inverse, 3, 5, batch=2, scale=1.5, transform=dfft.R2C) < 1e-12


def test_rc_line_matches_naive():
    """tests/emu_rc_pair.cpp: the R2C / C2R per-line steps of the interleaved z pass (one component per line) against a
    long-double DFT, Nz = 4..8192; rel-L2 <= 1e-15 (f64) / 1e-6 (f32)"""
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "emu")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "emu_rc_pair.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        print(r.stdout[-400:])
        assert r.returncode == 0 and "fails=0" in r.stdout, r.stdout[-2000:]


@pytest.mark.parametrize("inverse", [0, 1])
def test_interleaved_batch_and_scale(inverse):
    assert run_interleaved(4, SL, (8, 8, 64), 4, 1, P2P, inverse, 3, 3, batch=2, scale=0.375) < 1e-12
    assert run_interleaved(4, PE, (8, 8, 32), 2, 2, A2A, inverse, 3, 5, batch=2, scale=1.5) < 1e-12
    assert run_interleaved(1, SL, (64, 64, 64), 1, 1, P2P, inverse, 3, 3, batch=2) < 1e-12  # no batched stage


@pytest.mark.parametrize("inverse", [0, 1])
def test_slot_rule_catches_a_missing_rendezvous(inverse):
    """the replay's slot rule holds interleaved plans too: without the rendezvous of its transpositions, a pass reads a slot
    that a peer stored into"""
    assert run_interleaved(4, SL, (16, 8, 64), 4, 1, P2P, inverse, 3, 3) < 1e-12
    with pytest.raises(AssertionError, match="without a rendezvous"):
        run_interleaved(4, SL, (16, 8, 64), 4, 1, P2P, inverse, 3, 3, mutate=drop_rendezvous)


ONE = [(1, SL, (64, 64, 64), 1, 1, P2P), (1, SL, (512, 512, 512), 1, 1, P2P), (2, SL, (8, 8, 128), 2, 1, P2P),
       (4, ZY, (8, 4, 16), 4, 1, A2A), (8, PE, (16, 8, 16), 4, 2, A2A), (6, PE, (12, 9, 64), 3, 2, P2P)]


@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm", ONE)
@pytest.mark.parametrize("transform", [dfft.C2C, dfft.R2C])
def test_one_component_is_the_batched_plan(P, decomp, shape, p1, p2, comm, transform):
    """components = 1 describes byte for byte the schedules of dfft_plan_create_batched, in every direction and d"""
    if transform == dfft.R2C and any(n & (n - 1) for n in shape):
        pytest.skip("R2C plans take powers of two")
    for batch in (1, 2):
        for inverse in (0, 1):
            for d in (1, 2, 3):
                a = describe_batched(0, P, decomp, transform, shape, p1, p2, comm, SYNC, inverse, d, batch)
                b = describe_ilv(0, P, decomp, transform, shape, p1, p2, 1, batch, comm, inverse, d)
                assert json.dumps(a) == json.dumps(b)


def test_sizes_are_c_times_the_batched_plan():
    """domain size C times the batched plan's; work area: its slots of C times the largest domain over ranks, each rounded
    up to 256 bytes as every slot is"""
    cases = [(1, SL, (16, 8, 32), 1, 1, dfft.C2C), (4, PE, (12, 9, 64), 2, 2, dfft.C2C), (3, ZY, (6, 4, 16), 3, 1, dfft.C2C),
             (4, SL, (8, 8, 64), 4, 1, dfft.R2C), (6, PE, (16, 8, 64), 3, 2, dfft.R2C)]
    for P, decomp, shape, p1, p2, transform in cases:
        dom = []
        for r in range(P):
            rc, msg, comm, base = create(r, P, decomp, transform, shape, p1, p2, 1)
            assert rc == 0, msg
            dom.append(lib().dfft_get_domain_size(base))
            lib().dfft_plan_destroy(base)
            lib().dfft_comm_destroy(comm)
        nslots = describe_ilv(0, P, decomp, transform, shape, p1, p2, 3, 1, P2P, 0, 3)["nslots"]
        round256 = lambda b: (b + 255) // 256 * 256
        for r in range(P):
            rc, msg, comm, base = create(r, P, decomp, transform, shape, p1, p2, 1)
            assert rc == 0, msg
            rc, msg, comm2, plan = create(r, P, decomp, transform, shape, p1, p2, 3)
            assert rc == 0, msg
            assert lib().dfft_get_components(plan) == 3 and lib().dfft_get_components(base) == 1
            assert lib().dfft_get_domain_size(plan) == 3 * lib().dfft_get_domain_size(base)
            assert lib().dfft_get_work_size_device(base) == nslots * round256(max(dom))
            assert lib().dfft_get_work_size_device(plan) == nslots * round256(3 * max(dom))
            for fn in ("dfft_get_in_size", "dfft_get_out_size", "dfft_get_in_start", "dfft_get_out_start"):
                u, v = (C.c_size_t * 3)(), (C.c_size_t * 3)()
                check(getattr(lib(), fn)(plan, u))
                check(getattr(lib(), fn)(base, v))
                assert list(u) == list(v)
            for h, c in ((plan, comm2), (base, comm)):
                lib().dfft_plan_destroy(h)
                lib().dfft_comm_destroy(c)
    assert lib().dfft_get_components(None) == 0


def test_argument_validation():
    shape = (64, 64, 64)
    INVALID, UNSUPPORTED = -1, -5
    bad = [((SL, dfft.C2C, shape, 0), INVALID, "components"),
           ((SL, dfft.C2C, shape, 65), UNSUPPORTED, "64"),
           ((SL, dfft.R2C, (64, 64, 16384), 3), UNSUPPORTED, "8192"),
           ((SL, dfft.DCT, shape, 2), UNSUPPORTED, "C2C"),
           ((SL, dfft.C2C, (64, 64, 48), 2), UNSUPPORTED, "Nz"),
           ((SL, 7, shape, 2), INVALID, "transform")]
    for (decomp, transform, shp, comps), code, word in bad:
        rc, msg, comm, plan = create(0, 1, decomp, transform, shp, 1, 1, comps)
        assert rc == code and word in msg, (rc, msg)
        lib().dfft_comm_destroy(comm)
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, shape, 1, 1, 64)  # the largest C; Bluestein x, y are fine
    assert rc == 0, msg
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(comm)
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (48, 100, 64), 1, 1, 3)
    assert rc == 0, msg
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(comm)
    # batch x C overflow
    field = 64 ** 3 * 16 * 3
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, shape, 1, 1, 3, SIZE_MAX // field + 1)
    assert rc == -1 and "overflow" in msg
    lib().dfft_comm_destroy(comm)
    # kept axes
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, shape, 1, 1, 3)
    assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == UNSUPPORTED
    check(lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(1, 1, 1)))
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(comm)


def test_sequential_schedule_only():
    """no fused z + y stage at 512^3, no batched stage at 64^3, no overlapped schedule"""
    sc = describe_ilv(0, 1, SL, dfft.C2C, (512, 512, 512), 1, 1, 3, 1, P2P, 0, 3)
    assert [s["label"] for s in sc["steps"]] == ["z pass", "y pass", "x pass"] and sc["components"] == 3
    assert sc["steps"][0]["kind"] == ILV
    sc = describe_ilv(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, 2, 3, P2P, 1, 3)
    assert "batched pass" not in json.dumps(sc)


def test_python_binding_refusals():
    """the binding refuses the combinations it cannot express before it creates a plan (no device needed)"""
    p = dfft.MPIcuFFT_Slab.__new__(dfft.MPIcuFFT_Slab)
    p.config, p.precision, p.kinds, p.transform = dfft.Configurations(), dfft.F64, None, dfft.C2C
    p.comm = type("DryComm", (), {"size": 1, "_h": None})()
    for kw in ({"inplace": True}, {"spectral": (4, 4, 4)}, {"batch": 0}):
        with pytest.raises(ValueError):
            p.initFFT(dfft.GlobalSize(8, 8, 8), None, True, components=3, **kw)
    # batch 0 on the plain, in-place and per-axis-kind paths too
    for kinds, kw in ((None, {}), (None, {"inplace": True}), ((dfft.DCT, dfft.R2HC, dfft.DCT), {})):
        p.kinds = kinds
        with pytest.raises(ValueError):
            p.initFFT(dfft.GlobalSize(8, 8, 8), None, True, batch=0, **kw)
