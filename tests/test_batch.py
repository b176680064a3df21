"""Batched plans (dfft_plan_create_batched) without a GPU: argument checks, the batch = 1 identity, the selection of the
one-launch batched stage, its work list, and CPU replays of batched schedules.

The replay runs the step lists dfft_plan_describe returns for every rank of a batched plan through step_replay.py, on
distinct inputs per field.  Every field's block must match the oracle, and every step may only touch the caller's memory of
its own field (the per-field distance is the product of the buffer's layout, never the domain size)."""
import json
import os
import subprocess
import tempfile

import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import lib
from oracle import dft_oracle as O

from test_schedule_emulation import A2A, P2P, PE, SL, STREAMS, SYNC, ZY, describe

HERE = os.path.dirname(os.path.abspath(__file__))
SIZE_MAX = (1 << 64) - 1


def plan_of(P, decomp, transform, shape, p1, p2, batch, comm_method=P2P, send_method=SYNC, prec=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=dfft.F64 if prec is None else prec, comm=comm_method, send=send_method,
                  batch=batch)


def create(rank, P, decomp, transform, shape, p1, p2, batch, comm_method=P2P, send_method=SYNC, prec=None):
    """dry batched plan: (rc, message, comm, plan)"""
    return R.create(plan_of(P, decomp, transform, shape, p1, p2, batch, comm_method, send_method, prec), rank)


def describe_batched(rank, P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, batch, prec=None):
    return R.describe(plan_of(P, decomp, transform, shape, p1, p2, batch, comm_method, send_method, prec), rank, inverse, d)


def run_batched(P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, batch, prec=None):
    """Replays a batched exec on every rank on a distinct input per field; returns the worst rel-L2 error over all fields
    and ranks."""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    p = plan_of(P, decomp, transform, shape, p1, p2, batch, comm_method, send_method, prec)
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    if batch > 1:
        assert all(s["batch"] == batch for s in scheds)
    xs = [O.complex_input(shape, seed=1234 + f) if c2c else O.real_input(shape, seed=1234 + f) for f in range(batch)]
    specs = [O.fft_c2c(x, d) if c2c else O.fft_r2c(x, d) for x in xs]
    n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
    x, want = (specs, [n * x for x in xs]) if inverse else (xs, specs)
    return R.error(R.replay(p, inverse, d, x, scheds), want)


CASES = [
    # P, decomp, transform, shape, p1, p2, comm, send
    (1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC),          # blocked hand-over, one rank
    (1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC),
    (2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS),       # overlapped: streams join and fork again between fields
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, A2A, SYNC),
    (8, SL, dfft.R2C, (16, 8, 64), 8, 1, P2P, STREAMS),       # overlapped + blocked + tail column
    (4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, SYNC),         # blocked + tail (Nzc = 65)
    (4, ZY, dfft.R2C, (8, 4, 32), 4, 1, P2P, SYNC),
    (4, ZY, dfft.C2C, (8, 4, 16), 4, 1, A2A, SYNC),
    (8, PE, dfft.R2C, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 16), 4, 2, A2A, SYNC),
    (4, PE, dfft.C2C, (8, 8, 128), 2, 2, P2P, STREAMS),       # overlapped pencil forward
]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_batched_schedules(P, decomp, transform, shape, p1, p2, comm, send, inverse):
    assert run_batched(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_batched_partial_schedules(d, inverse, comm):
    assert run_batched(8, PE, dfft.R2C, (8, 16, 32), 2, 4, comm, SYNC, inverse, d, 2) < 1e-12
    assert run_batched(4, PE, dfft.C2C, (8, 8, 16), 2, 2, comm, SYNC, inverse, d, 3) < 1e-12


def test_batched_overlapped_pencil_inverse(monkeypatch):
    """the overlapped pencil inverse (selected by dfft_plan_tune, built directly with DFFT_PENCIL_OVERLAP=2)"""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    for inverse in (0, 1):
        assert run_batched(4, PE, dfft.R2C, (8, 16, 128), 2, 2, P2P, STREAMS, inverse, 3, 2) < 1e-12


@pytest.mark.parametrize("shape,batch,prec", [((32, 32, 32), 3, dfft.F64), ((64, 64, 64), 2, dfft.F64), ((32, 32, 32), 2, dfft.F32)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_batched_stage_replay(shape, batch, prec, inverse):
    """the one-launch stage, listed as its three views over all fields, against the oracle"""
    sc = describe_batched(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec)
    assert [s["field"] for s in sc["steps"]] == [-1, -1, -1]
    assert run_batched(1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec) < 1e-12


def _labels(shape, batch, inverse=0, prec=dfft.F64, transform=dfft.C2C, P=1):
    sc = describe_batched(0, P, SL, transform, shape, P, 1, P2P, SYNC, inverse, 3, batch, prec)
    return [s["label"] for s in sc["steps"]]


def test_selection_of_the_batched_stage():
    """one launch for two or more cubic 32^3 / 64^3 complex fields on one rank, in both precisions; the per-field schedule
    otherwise"""
    one = ["batched pass: z lines", "batched pass: y lines", "batched pass: x lines"]
    for n in (32, 64):
        for prec in (dfft.F64, dfft.F32):
            assert _labels((n, n, n), 2, 0, prec) == one
            assert _labels((n, n, n), 64, 1, prec) == one[::-1]
            assert _labels((n, n, n), 1, 0, prec) == ["z pass", "y pass", "x pass"]
    per_field = lambda labels, b: labels == ["z pass", "y pass", "x pass"] * b
    assert per_field(_labels((128, 128, 128), 2), 2)      # larger fields
    assert per_field(_labels((16, 16, 16), 2), 2)         # length not instantiated
    assert per_field(_labels((64, 64, 32), 2), 2)         # not cubic
    assert _labels((64, 64, 64), 2, transform=dfft.R2C)[0] == "z pass (R2C)"
    assert "batched pass" not in " ".join(_labels((64, 64, 64), 2, P=2))
    sc = describe_batched(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, P2P, SYNC, 0, 2, 2)  # partial transforms: per field
    assert [s["field"] for s in sc["steps"]] == [0, 0, 1, 1]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES + [(1, SL, dfft.C2C, (64, 64, 64), 1, 1, P2P, SYNC)])
def test_batch_one_is_the_unbatched_plan(P, decomp, transform, shape, p1, p2, comm, send):
    """dfft_plan_create_batched(batch = 1) describes byte for byte the schedules of dfft_plan_create"""
    for inverse in (0, 1):
        a = describe(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, 3)
        b = describe_batched(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, 1)
        assert json.dumps(a) == json.dumps(b)


def test_batch_argument_validation():
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, 0)
    assert rc == -1 and "batch" in msg
    lib().dfft_comm_destroy(comm)
    field = 64 ** 3 * 16
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, SIZE_MAX // field + 1)
    assert rc == -1 and "overflow" in msg
    lib().dfft_comm_destroy(comm)
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, SIZE_MAX // field)
    assert rc == 0, msg
    assert lib().dfft_get_batch(plan) == SIZE_MAX // field
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(comm)
    # R2C: the widest buffer is the complex side of the partial transforms
    rc, msg, comm, plan = create(0, 1, SL, dfft.R2C, (64, 64, 64), 1, 1, SIZE_MAX // (64 * 64 * 33 * 16) + 1)
    assert rc == -1 and "overflow" in msg
    lib().dfft_comm_destroy(comm)
    assert lib().dfft_get_batch(None) == 0


def test_work_list():
    """the field-ordered work list of the batched stage and the launch decoding of a captured / replayed launch"""
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "batch_order_test")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "batch_order_test.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0 and "fails=0" in r.stdout, r.stdout[-2000:]
