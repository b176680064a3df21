"""C2C plans with axis lengths that are not powers of two, without a GPU: length validation, the step lists (Bluestein
passes carry "n", their "log2n" is log2 M) and CPU replays of every rank's step list on 1-8 ranks.

The replay (step_replay.py) runs the geometry-only plans' step lists in lock step with numpy FFTs of the length each pass
names ("n" when present, else 2^log2n; "n" only on lengths that are not powers of two, with log2n = log2 M, M >= 2n - 1 >
M / 2), multiplies the stores of each step by its "scale", checks the happens-before order of every access, and compares
every rank's output with the oracle (times the scale)."""
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import lib
from oracle import dft_oracle as O

from test_batch import create
from test_schedule_emulation import describe

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
DFFT_ERR_UNSUPPORTED = -5


def plan_of(P, decomp, shape, p1, p2, comm, send, batch=1, scale=None, transform=dfft.C2C):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, comm=comm, send=send, batch=batch, scale=scale)


def describe_plan(rank, P, decomp, shape, p1, p2, comm, send, inverse, d, batch=1, scale=None, transform=dfft.C2C):
    return R.describe(plan_of(P, decomp, shape, p1, p2, comm, send, batch, scale, transform), rank, inverse, d)


def replay(P, decomp, shape, p1, p2, comm, send, inverse, d, batch=1, s=1.0):
    """worst rel-L2 error of every rank's output against the oracle times s"""
    nx, ny, nz = shape
    p = plan_of(P, decomp, shape, p1, p2, comm, send, batch, None if s == 1.0 else (1.0, s) if inverse else (s, 1.0))
    scheds = [R.describe(p, r, inverse, d) for r in range(P)]
    for sc in scheds:
        assert not sc["overlapped"]
        assert all(st.get("n", 1 << st.get("log2n", 0)) in shape for st in sc["steps"] if st["type"] == 0)
    xs = [O.complex_input(shape, seed=31 + f) for f in range(batch)]
    specs = [O.fft_c2c(x, d) for x in xs]
    n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
    x, want = (specs, [s * n * x for x in xs]) if inverse else (xs, [s * sp for sp in specs])
    return R.error(R.replay(p, inverse, d, x, scheds), want)


CASES = [
    # P, decomp, shape, p1, p2, comm, send
    (1, SL, (12, 10, 7), 1, 1, P2P, SYNC),
    (1, SL, (3, 5, 7), 1, 1, P2P, SYNC),
    (1, SL, (6, 100, 130), 1, 1, P2P, SYNC),      # one rank, blocked hand-over (CH = 32) with a tail of 2 columns
    (2, SL, (6, 100, 130), 2, 1, P2P, SYNC),      # blocked hand-over with tails, peer stores
    (5, SL, (96, 20, 12), 5, 1, P2P, SYNC),       # 96 over 5
    (3, SL, (100, 9, 6), 3, 1, A2A, SYNC),        # 100 over 3
    (4, SL, (16, 12, 96), 4, 1, P2P, STREAMS),    # Streams: sequential schedule
    (1, ZY, (6, 12, 7), 1, 1, P2P, SYNC),
    (2, ZY, (6, 5, 7), 2, 1, P2P, SYNC),          # 7 over 2
    (3, ZY, (12, 10, 7), 3, 1, A2A, SYNC),
    (1, PE, (6, 10, 7), 1, 1, P2P, SYNC),
    (6, PE, (12, 10, 7), 2, 3, P2P, SYNC),
    (8, PE, (12, 10, 9), 4, 2, A2A, SYNC),
    (4, PE, (5, 96, 24), 2, 2, P2P, SYNC),        # mixed: power-of-two and other axes
]


@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_nonpow2_schedules(P, decomp, shape, p1, p2, comm, send, inverse):
    assert replay(P, decomp, shape, p1, p2, comm, send, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_nonpow2_partial(d, inverse, comm):
    assert replay(6, PE, (12, 10, 7), 2, 3, comm, SYNC, inverse, d) < 1e-12
    assert replay(1, PE, (6, 10, 7), 1, 1, comm, SYNC, inverse, d) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_nonpow2_batch_and_scale(inverse):
    """batch 2 and a scale that is not 1: every output value is scaled exactly once"""
    assert replay(1, SL, (12, 10, 7), 1, 1, P2P, SYNC, inverse, 3, batch=2) < 1e-12
    assert replay(1, SL, (12, 10, 7), 1, 1, P2P, SYNC, inverse, 3, batch=2, s=3.0) < 1e-12
    assert replay(2, SL, (6, 100, 130), 2, 1, P2P, SYNC, inverse, 3, batch=2, s=3.0) < 1e-12
    assert replay(4, PE, (6, 10, 7), 2, 2, A2A, SYNC, inverse, 2, batch=2, s=0.3) < 1e-12


def _dry(shape, transform=dfft.C2C, P=1, decomp=SL, p1=1, p2=1, send=SYNC):
    rc, msg, c, plan = create(0, P, decomp, transform, shape, p1, p2, 1, P2P, send)
    if rc == 0:
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return rc, msg


def test_length_validation():
    assert _dry((96, 100, 7))[0] == 0
    assert _dry((4096, 3, 5))[0] == 0
    assert _dry((8192, 8192, 4095))[0] == 0
    for bad in ((4097, 8, 8), (8, 1, 8), (8, 8, 1), (6000, 8, 8), (8, 8, 16384)):
        rc, msg = _dry(bad)
        assert rc == DFFT_ERR_UNSUPPORTED and "C2C" in msg, bad
    rc, msg = _dry((96, 64, 64), dfft.R2C)
    assert rc == DFFT_ERR_UNSUPPORTED and "powers of two" in msg
    rc, msg = _dry((64, 64, 96), dfft.R2C)
    assert rc == DFFT_ERR_UNSUPPORTED and "powers of two" in msg


def test_streams_plans_run_the_sequential_schedule():
    """a Streams plan with an axis that is not a power of two builds the sequential schedule (the same plan with
    power-of-two axes builds the overlapped one)"""
    for inverse in (0, 1):
        assert describe(0, 4, SL, dfft.C2C, (16, 16, 64), 4, 1, P2P, STREAMS, inverse, 3)["overlapped"]
        assert not describe(0, 4, SL, dfft.C2C, (16, 12, 64), 4, 1, P2P, STREAMS, inverse, 3)["overlapped"]
    assert describe(0, 8, PE, dfft.C2C, (16, 32, 256), 2, 4, P2P, STREAMS, 0, 3)["overlapped"]
    assert not describe(0, 8, PE, dfft.C2C, (16, 32, 96), 2, 4, P2P, STREAMS, 0, 3)["overlapped"]


@pytest.mark.parametrize("shape", [(32, 32, 32), (64, 64, 64), (256, 256, 256), (512, 512, 512)])
def test_power_of_two_descriptions_have_no_length_key(shape):
    """power-of-two plans (including those of the fused and batched stages) carry no "n" key"""
    for inverse in (0, 1):
        for batch in (1, 2):
            sc = describe_plan(0, 1, SL, shape, 1, 1, P2P, SYNC, inverse, 3, batch)
            assert all("n" not in st for st in sc["steps"])


def test_fused_and_batched_stages_are_not_chosen():
    """the fused z + y stage and the one-launch batched stage need power-of-two lengths: a 384^3 plan, larger than the
    L2, runs three standalone passes, and a batch of 48^3 fields runs its per-field schedule"""
    for inverse in (0, 1):
        labels = [st["label"] for st in describe_plan(0, 1, SL, (384, 384, 384), 1, 1, P2P, SYNC, inverse, 3)["steps"]]
        assert set(labels) == {"z pass", "y pass", "x pass", "y pass (tail)", "x pass (tail)"}  # blocked hand-over, CH = 10
        steps = describe_plan(0, 1, SL, (48, 48, 48), 1, 1, P2P, SYNC, inverse, 3, batch=4)["steps"]
        assert len(steps) == 12 and all(st["n"] == 48 for st in steps)
