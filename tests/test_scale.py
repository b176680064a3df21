"""Output scale (dfft_plan_set_scale) without a GPU: argument checks and defaults, the step list of scaled plans, and CPU
replays that prove every output value is scaled exactly once.

A scaled plan's dfft_plan_describe must equal the unscaled one except for a "scale" key on the steps whose stores are
final.  The replay runs the scaled step lists of every rank through step_replay.py, which multiplies each step's stores
by its "scale" and counts how often each output value is scaled, and compares every rank's output with the oracle times
the scale: a value scaled twice or not at all is off by that factor."""
import ctypes as C
import json
import math
from dataclasses import replace

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import lib
from oracle import dft_oracle as O

from test_batch import create
from test_schedule_emulation import A2A, P2P, PE, SL, STREAMS, SYNC, ZY

S = 3.0  # a scale that no double application or omission can hide


def plan_of(P, decomp, transform, shape, p1, p2, comm, send, batch=1, prec=None, scale=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=dfft.F64 if prec is None else prec, comm=comm, send=send, batch=batch,
                  scale=scale)


def describe_scaled(rank, P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, prec=None, scale=None):
    return R.describe_text(plan_of(P, decomp, transform, shape, p1, p2, comm, send, batch, prec, scale), rank, inverse, d)


def run_scaled(P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, prec=None):
    """Replays the scaled exec (scale S in the direction under test) on every rank; returns the worst rel-L2 error of the
    output against S times the oracle.  Also checks that the scaled step lists differ from the unscaled ones only by the
    "scale" key of the steps that write the caller's output last."""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    p = plan_of(P, decomp, transform, shape, p1, p2, comm, send, batch, prec, (1.0, S) if inverse else (S, 1.0))
    scheds = []
    for r in range(P):
        a, b = R.describe(replace(p, scale=None), r, inverse, d), R.describe(p, r, inverse, d)
        marked = [k for k, st in enumerate(b["steps"]) if "scale" in st]
        assert marked and all(b["steps"][k]["scale"] == S for k in marked)
        assert a == {**b, "steps": [{key: v for key, v in st.items() if key != "scale"} for st in b["steps"]]}
        # marked: the steps that store into the caller's output with no later step of the same field reading it
        for k, st in enumerate(a["steps"]):
            later_read = any(t.get("in_user") == 2 and t.get("field", 0) == st.get("field", 0) for t in a["steps"][k + 1:])
            assert (k in marked) == (st["type"] == 0 and st["out_user"] == 2 and not later_read), (k, st["label"])
        scheds.append(b)
    xs = [O.complex_input(shape, seed=99 + f) if c2c else O.real_input(shape, seed=99 + f) for f in range(batch)]
    specs = [O.fft_c2c(x, d) if c2c else O.fft_r2c(x, d) for x in xs]
    n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
    x, want = (specs, [S * n * x for x in xs]) if inverse else (xs, [S * s for s in specs])
    return R.error(R.replay(p, inverse, d, x, scheds), want)


CASES = [
    # P, decomp, transform, shape, p1, p2, comm, send
    (1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC),          # blocked hand-over, one rank
    (1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC),
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P, SYNC),          # peer stores
    (3, SL, dfft.R2C, (8, 16, 16), 3, 1, P2P, SYNC),          # uneven split
    (8, SL, dfft.C2C, (16, 16, 64), 8, 1, A2A, SYNC),
    (4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, SYNC),         # blocked + tail column (Nzc = 65)
    (8, SL, dfft.R2C, (16, 8, 64), 8, 1, P2P, STREAMS),       # overlapped + blocked + tail
    (8, SL, dfft.C2C, (32, 16, 256), 8, 1, P2P, STREAMS),     # overlapped + blocked
    (2, SL, dfft.C2C, (8, 8, 128), 2, 1, A2A, STREAMS),
    (1, ZY, dfft.C2C, (8, 8, 16), 1, 1, P2P, SYNC),
    (4, ZY, dfft.R2C, (8, 4, 32), 4, 1, P2P, SYNC),
    (4, ZY, dfft.C2C, (8, 4, 16), 4, 1, A2A, SYNC),
    (1, PE, dfft.C2C, (8, 8, 16), 1, 1, P2P, SYNC),
    (8, PE, dfft.R2C, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 16), 4, 2, A2A, SYNC),
    (8, PE, dfft.R2C, (16, 16, 2048), 4, 2, P2P, SYNC),       # blocked second transposition with tail columns
]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("batch", [1, 3])
def test_scaled_schedules(P, decomp, transform, shape, p1, p2, comm, send, inverse, batch):
    assert run_scaled(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, batch) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
@pytest.mark.parametrize("batch", [1, 3])
def test_scaled_partial_schedules(d, inverse, comm, batch):
    assert run_scaled(8, PE, dfft.R2C, (8, 16, 32), 2, 4, comm, SYNC, inverse, d, batch) < 1e-12
    assert run_scaled(4, PE, dfft.C2C, (8, 8, 16), 2, 2, comm, SYNC, inverse, d, batch) < 1e-12
    assert run_scaled(1, PE, dfft.C2C, (8, 8, 16), 1, 1, comm, SYNC, inverse, d, batch) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_scaled_overlapped_pencil(inverse, monkeypatch):
    """overlapped pencil schedules, built without the plan-time measurement that selects the inverse one"""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    for batch in (1, 3):
        assert run_scaled(8, PE, dfft.C2C, (16, 32, 256), 2, 4, P2P, STREAMS, inverse, 3, batch) < 1e-12
        assert run_scaled(4, PE, dfft.R2C, (8, 16, 128), 2, 2, P2P, STREAMS, inverse, 3, batch) < 1e-12


@pytest.mark.parametrize("env", [{"DFFT_OVL_GROUPS": "1", "DFFT_OVL_CHUNKS": "8"}, {"DFFT_OVL_GROUPS": "2", "DFFT_OVL_CHUNKS": "2"}])
@pytest.mark.parametrize("inverse", [0, 1])
def test_scaled_overlap_chunks(env, inverse, monkeypatch):
    """every z chunk of the overlapped x pass stores final values (the chunkings dfft_plan_tune chooses between)"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert run_scaled(8, SL, dfft.C2C, (32, 16, 512), 8, 1, P2P, STREAMS, inverse, 3) < 1e-12
    assert run_scaled(4, SL, dfft.R2C, (16, 16, 1024), 4, 1, P2P, STREAMS, inverse, 3) < 1e-12


@pytest.mark.parametrize("shape,batch,prec", [((512, 256, 256), 1, dfft.F64), ((256, 256, 256), 1, dfft.F32),
                                              ((32, 32, 32), 3, dfft.F64), ((64, 64, 64), 2, dfft.F32)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_scaled_fused_and_batched_stages(shape, batch, prec, inverse):
    """the fused z + y stage (listed as its two phases) and the one-launch batched stage (its three views): only the
    last phase is scaled"""
    plain = json.loads(describe_scaled(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec))
    scaled = json.loads(describe_scaled(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec, (0.3, 0.3)))
    labels = [s["label"] for s in plain["steps"]]
    marked = [s["label"] for s in scaled["steps"] if "scale" in s]
    want = 0.3 if prec == dfft.F64 else float(np.float32(0.3))
    assert all(s["scale"] == want for s in scaled["steps"] if "scale" in s)
    if batch > 1:
        assert marked == ["batched pass: z lines" if inverse else "batched pass: x lines"] and len(labels) == 3
    elif inverse:
        assert labels == ["x pass", "yz pass: y phase", "yz pass: z phase"] and marked == ["yz pass: z phase"]
    else:
        assert "zy pass: z phase" in labels and marked == ["x pass"]
    if shape[0] <= 64:
        assert run_scaled(1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec) < 1e-12


def test_defaults_and_validation():
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, 1)
    assert rc == 0, msg
    f, i = C.c_double(), C.c_double()
    assert lib().dfft_plan_get_scale(plan, C.byref(f), C.byref(i)) == 0 and (f.value, i.value) == (1.0, 1.0)
    for bad in (math.nan, math.inf, -math.inf):
        assert lib().dfft_plan_set_scale(plan, bad, 1.0) == -1
        assert lib().dfft_plan_set_scale(plan, 1.0, bad) == -1
    assert lib().dfft_plan_get_scale(plan, C.byref(f), C.byref(i)) == 0 and (f.value, i.value) == (1.0, 1.0)
    assert lib().dfft_plan_set_scale(plan, 0.0, -2.5) == 0  # zero and negative scales are finite
    assert lib().dfft_plan_get_scale(plan, C.byref(f), C.byref(i)) == 0 and (f.value, i.value) == (0.0, -2.5)
    assert lib().dfft_plan_get_scale(plan, None, None) == 0
    assert lib().dfft_plan_set_scale(None, 1.0, 1.0) == -1
    assert lib().dfft_plan_get_scale(None, C.byref(f), C.byref(i)) == -1
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES[:8] + CASES[12:14])
def test_unit_scale_is_byte_identical(P, decomp, transform, shape, p1, p2, comm, send):
    """(1, 1), and a scale set back to (1, 1), describe exactly the plan without a scale; a scale of one direction leaves
    the other direction's description alone"""
    for inverse in (0, 1):
        for d in (1, 3):
            ref = describe_scaled(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, d)
            assert describe_scaled(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, d, scale=(1.0, 1.0)) == ref
            other = (1.0, 0.5) if not inverse else (0.5, 1.0)
            assert describe_scaled(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, d, scale=other) == ref
    rc, msg, c, plan = create(0, P, decomp, transform, shape, p1, p2, 1, comm, send)
    assert rc == 0, msg
    need = C.c_size_t()
    texts = []
    for sc in ((1.0, 1.0), (0.25, 4.0), (1.0, 1.0)):
        assert lib().dfft_plan_set_scale(plan, *sc) == 0
        assert lib().dfft_plan_describe(plan, 1, 3, None, 0, C.byref(need)) == 0
        buf = C.create_string_buffer(need.value)
        assert lib().dfft_plan_describe(plan, 1, 3, buf, need.value, C.byref(need)) == 0
        texts.append(buf.value)
    assert texts[0] == texts[2] != texts[1]
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
