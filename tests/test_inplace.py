"""In-place plans (dfft_plan_create_inplace) without a GPU: argument checks, the work area, and CPU replays of every rank's
step list with the caller's `in` and `out` mapped to ONE address range (step_replay.py).

The buffer of a rank holds `batch` fields dfft_get_domain_size() bytes apart; real rows of R2C / C2R plans are padded to
Nz/2 + 1 complex units, and the padding must never be read or written.  The replay's happens-before check sees the
read-after-write and write-after-read pairs on the buffer, its line check that a line only writes addresses that it reads
itself or that no other line of the step reads (the passes load a line or tile completely before they store it, so that is
what in place needs), and its phase check that the two phases of the fused z + y stage and of the one-launch batched
stage, which run concurrently, touch disjoint planes / fields."""
import ctypes as C

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import check, lib
from oracle import dft_oracle as O

from test_schedule_emulation import A2A, P2P, PE, SL, STREAMS, SYNC, ZY

SIZE_MAX = (1 << 64) - 1


def plan_of(P, decomp, transform, shape, p1, p2, batch=1, comm=P2P, send=SYNC, prec=None, scale=None, inplace=True):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=dfft.F64 if prec is None else prec, comm=comm, send=send, batch=batch,
                  inplace=inplace, scale=scale)


def create(rank, P, decomp, transform, shape, p1, p2, batch=1, comm=P2P, send=SYNC, prec=None, inplace=True):
    """dry plan: (rc, message, comm, plan)"""
    return R.create(plan_of(P, decomp, transform, shape, p1, p2, batch, comm, send, prec, inplace=inplace), rank)


def describe(rank, P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, prec=None, scale=None, inplace=True):
    return R.describe(plan_of(P, decomp, transform, shape, p1, p2, batch, comm, send, prec, scale, inplace), rank, inverse, d)


def run_inplace(P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, scale=1.0, prec=None, mutate=None):
    """Replays an in-place exec on every rank; returns the worst rel-L2 error of the output against scale times the
    oracle."""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    sc_ = None if scale == 1.0 else ((1.0, scale) if inverse else (scale, 1.0))
    p = plan_of(P, decomp, transform, shape, p1, p2, batch, comm, send, prec, sc_)
    xs = [O.complex_input(shape, seed=77 + f) if c2c else O.real_input(shape, seed=77 + f) for f in range(batch)]
    specs = [O.fft_c2c(x, d) if c2c else O.fft_r2c(x, d) for x in xs]
    n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
    x, want = (specs, [scale * n * x for x in xs]) if inverse else (xs, [scale * s for s in specs])
    return R.error(R.replay(p, inverse, d, x, mutate=mutate), want)


# ---- argument checks ------------------------------------------------------------------------------------------------
def _plan_info(P, decomp, transform, shape, p1, p2, inplace, batch=1, comm=P2P):
    rc, msg, c, plan = create(0, P, decomp, transform, shape, p1, p2, batch, comm, SYNC, None, inplace)
    assert rc == 0, msg
    info = dict(inplace=lib().dfft_plan_is_inplace(plan), work=lib().dfft_get_work_size_device(plan), dom=lib().dfft_get_domain_size(plan))
    in_size = (C.c_size_t * 3)()
    out_size = (C.c_size_t * 3)()
    check(lib().dfft_get_in_size(plan, in_size))
    check(lib().dfft_get_out_size(plan, out_size))
    info["in_size"], info["out_size"] = list(in_size), list(out_size)
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return info


def test_is_inplace():
    assert _plan_info(1, SL, dfft.C2C, (8, 8, 8), 1, 1, True)["inplace"] == 1
    assert _plan_info(1, SL, dfft.C2C, (8, 8, 8), 1, 1, False)["inplace"] == 0
    assert lib().dfft_plan_is_inplace(None) == 0


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm", [
    (1, SL, dfft.C2C, (64, 32, 16), 1, 1, P2P), (1, ZY, dfft.R2C, (16, 8, 32), 1, 1, P2P), (1, PE, dfft.C2C, (8, 16, 32), 1, 1, P2P),
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P), (4, SL, dfft.R2C, (16, 8, 64), 4, 1, A2A), (6, PE, dfft.R2C, (8, 16, 16), 3, 2, A2A),
    (4, ZY, dfft.C2C, (8, 4, 16), 4, 1, P2P)])
def test_work_area(P, decomp, transform, shape, p1, p2, comm):
    """one rank: one slot, half the out-of-place work area; several ranks: the out-of-place slots"""
    ip = describe(0, P, decomp, transform, shape, p1, p2, comm, SYNC, 0, 3)
    oop = describe(0, P, decomp, transform, shape, p1, p2, comm, SYNC, 0, 3, inplace=False)
    assert ip["inplace"] is True and "inplace" not in oop
    assert ip["slot_bytes"] == oop["slot_bytes"] and ip["domain_bytes"] == oop["domain_bytes"]
    if P == 1:
        assert ip["nslots"] == 1 and oop["nslots"] == 2
        assert ip["work_bytes"] == ip["slot_bytes"] == oop["work_bytes"] // 2
    else:
        assert ip["nslots"] == oop["nslots"] >= 2 and ip["work_bytes"] == oop["work_bytes"]


@pytest.mark.parametrize("P,decomp,shape,p1,p2", [(1, SL, (8, 16, 64), 1, 1), (3, SL, (8, 16, 16), 3, 1), (4, ZY, (8, 4, 32), 4, 1),
                                                  (6, PE, (8, 16, 16), 3, 2), (8, PE, (16, 16, 2048), 4, 2), (2, PE, (4, 4, 4), 1, 2)])
def test_domain_covers_the_padded_input(P, decomp, shape, p1, p2):
    """dfft_get_domain_size covers the padded real input ([X][Y][Nz/2+1] complex units) and every other layout of every
    rank; the getters keep the logical sizes"""
    nzc = shape[2] // 2 + 1
    for r in range(P):
        rc, msg, c, plan = create(r, P, decomp, dfft.R2C, shape, p1, p2)
        assert rc == 0, msg
        dom = lib().dfft_get_domain_size(plan)
        in_size = (C.c_size_t * 3)()
        check(lib().dfft_get_in_size(plan, in_size))
        assert in_size[2] == shape[2]
        assert dom >= in_size[0] * in_size[1] * nzc * 16
        for w in (1, 2, 3):
            assert dom >= int(np.prod(dfft.layout(decomp, dfft.R2C, *shape, p1, p2, r, w)[0])) * 16
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)


def test_batch_validation():
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, batch=0)
    assert rc == -1 and "batch" in msg
    lib().dfft_comm_destroy(c)
    # a field is domain_size = 8^3 * 16 bytes: one field too many overflows size_t
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, batch=SIZE_MAX // (8 ** 3 * 16) + 1)
    assert rc == -1 and "overflows" in msg
    lib().dfft_comm_destroy(c)
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, batch=SIZE_MAX // (8 ** 3 * 16))
    assert rc == 0, msg
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    # R2C: the padded input of an in-place plan is larger than the logical one
    rc, msg, c, plan = create(0, 1, SL, dfft.R2C, (8, 8, 8), 1, 1, batch=SIZE_MAX // (8 * 8 * 5 * 16) + 1)
    assert rc == -1 and "overflows" in msg
    lib().dfft_comm_destroy(c)


def test_step_lists_mark_the_buffer():
    """one rank, forward: the z pass runs in place in the buffer, the y pass reads it into the slot, the x pass writes it
    back; inverse: x pass buffer -> slot, y pass slot -> buffer, z pass in place"""
    fwd = describe(0, 1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3)["steps"]
    assert [(s["label"], s["in_user"], s["out_user"]) for s in fwd] == [("z pass", 1, 2), ("y pass", 2, 0), ("x pass", 0, 2)]
    inv = describe(0, 1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 1, 3)["steps"]
    assert [(s["label"], s["in_user"], s["out_user"]) for s in inv] == [("x pass", 1, 0), ("y pass", 0, 2), ("z pass", 2, 2)]
    # padded real rows: R2C input lines and C2R output lines are Nz/2 + 1 complex units apart
    r2c = describe(0, 1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC, 0, 3)["steps"][0]
    assert r2c["kind"] == 2 and r2c["in"]["segs"][0]["sA1"] == 129 and r2c["out"]["segs"][0]["sA1"] == 129
    c2r = describe(0, 1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC, 1, 3)["steps"][-1]
    assert c2r["kind"] == 3 and c2r["in"]["segs"][0]["sA1"] == 129 and c2r["out"]["segs"][0]["sA1"] == 129
    # the scale is on the steps that store the final values only
    sc = describe(0, 1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3, scale=(0.5, 1.0))["steps"]
    assert ["scale" in s for s in sc] == [False, False, True]


# ---- replays --------------------------------------------------------------------------------------------------------
CASES = [
    # P, decomp, transform, shape, p1, p2, comm, send
    (1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC),          # blocked hand-over, one slot
    (1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC),          # padded rows, blocked + tail column
    (1, ZY, dfft.C2C, (8, 8, 16), 1, 1, P2P, SYNC),
    (1, ZY, dfft.R2C, (8, 4, 32), 1, 1, P2P, SYNC),
    (1, PE, dfft.C2C, (8, 8, 16), 1, 1, P2P, SYNC),
    (1, PE, dfft.R2C, (8, 16, 64), 1, 1, P2P, SYNC),
    (2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS),       # overlapped slab
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P, SYNC),
    (3, SL, dfft.R2C, (8, 16, 16), 3, 1, P2P, SYNC),          # uneven split
    (3, SL, dfft.R2C, (16, 16, 64), 3, 1, P2P, STREAMS),      # uneven, overlapped, tail column
    (8, SL, dfft.C2C, (16, 16, 64), 8, 1, A2A, SYNC),
    (8, SL, dfft.R2C, (16, 8, 64), 8, 1, P2P, STREAMS),       # overlapped + blocked + tail
    (4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, SYNC),         # blocked + tail column (Nzc = 65)
    (4, ZY, dfft.R2C, (8, 4, 32), 4, 1, P2P, SYNC),
    (3, ZY, dfft.C2C, (8, 4, 16), 3, 1, A2A, SYNC),
    (8, PE, dfft.R2C, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 16), 4, 2, A2A, SYNC),
    (6, PE, dfft.R2C, (8, 16, 16), 3, 2, P2P, SYNC),          # uneven
    (8, PE, dfft.R2C, (16, 16, 2048), 4, 2, P2P, SYNC),       # blocked second transposition with tail columns
]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("batch", [1, 3])
def test_inplace_schedules(P, decomp, transform, shape, p1, p2, comm, send, inverse, batch):
    assert run_inplace(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, batch) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_inplace_partial(d, inverse, comm):
    assert run_inplace(8, PE, dfft.R2C, (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert run_inplace(4, PE, dfft.C2C, (8, 8, 16), 2, 2, comm, SYNC, inverse, d, batch=3) < 1e-12
    assert run_inplace(1, PE, dfft.R2C, (8, 8, 16), 1, 1, comm, SYNC, inverse, d) < 1e-12
    assert run_inplace(1, PE, dfft.C2C, (8, 8, 16), 1, 1, comm, SYNC, inverse, d, batch=3, scale=3.0) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_scale(inverse):
    """a scale that is not 1 lands on every output value exactly once, also where the buffer holds intermediates"""
    assert run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, batch=3, scale=3.0) < 1e-12
    assert run_inplace(1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC, inverse, 3, scale=0.25) < 1e-12
    assert run_inplace(3, SL, dfft.R2C, (16, 16, 64), 3, 1, P2P, STREAMS, inverse, 3, batch=3, scale=3.0) < 1e-12
    assert run_inplace(6, PE, dfft.R2C, (8, 16, 16), 3, 2, A2A, SYNC, inverse, 3, scale=3.0) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_overlapped_pencil(inverse, monkeypatch):
    """overlapped pencil schedules, built without the plan-time measurement that selects the inverse one"""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    assert run_inplace(8, PE, dfft.C2C, (16, 32, 256), 2, 4, P2P, STREAMS, inverse, 3) < 1e-12
    assert run_inplace(4, PE, dfft.R2C, (8, 16, 128), 2, 2, P2P, STREAMS, inverse, 3, batch=3) < 1e-12
    assert run_inplace(8, PE, dfft.R2C, (16, 16, 2048), 4, 2, P2P, STREAMS, inverse, 3) < 1e-12


@pytest.mark.parametrize("shape,batch,prec", [((256, 256, 256), 1, dfft.F64), ((512, 256, 256), 1, dfft.F32), ((32, 32, 32), 3, dfft.F64),
                                              ((64, 64, 64), 2, dfft.F32)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_fused_and_batched_stages(shape, batch, prec, inverse):
    """the fused z + y stage in place (forward: phase A z lines in place, phase B y tiles into the slot; inverse: phase A
    y tiles into the buffer, phase B z lines in place) and the one-launch batched stage with in == out"""
    sc = describe(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec)
    labels = [(s["label"], s["in_user"], s["out_user"]) for s in sc["steps"]]
    if batch > 1:
        assert labels == ([("batched pass: x lines", 1, 2), ("batched pass: y lines", 2, 2), ("batched pass: z lines", 2, 2)] if inverse else
                          [("batched pass: z lines", 1, 2), ("batched pass: y lines", 2, 2), ("batched pass: x lines", 2, 2)])
    elif inverse:
        assert labels == [("x pass", 1, 0), ("yz pass: y phase", 0, 2), ("yz pass: z phase", 2, 2)]
    else:
        assert labels == [("zy pass: z phase", 1, 2), ("zy pass: y phase", 2, 0), ("x pass", 0, 2)]
    if shape[0] <= 64 or shape == (256, 256, 256):
        assert run_inplace(1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, scale=0.5, prec=prec) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_bluestein(inverse):
    """a shape with lengths that are not powers of two (Bluestein passes, sequential schedule)"""
    assert run_inplace(1, SL, dfft.C2C, (12, 10, 7), 1, 1, P2P, SYNC, inverse, 3, batch=2, scale=3.0) < 1e-12
    assert run_inplace(3, PE, dfft.C2C, (12, 10, 7), 3, 1, A2A, SYNC, inverse, 3) < 1e-12


def _shift_rows(label):
    """schedule mutation: the in-place pass `label` stores every line one row further on (into the next line's input)"""
    def mutate(scheds):
        for sc in scheds:
            for st in sc["steps"]:
                if st["type"] == 0 and st["label"] == label:
                    seg = st["out"]["segs"][0]
                    seg["base"] += seg["sA1"] * sc["esize"]
    return mutate


def test_line_check_catches_cross_line_writes():
    """the line check is not vacuous: a z pass that stores each line into the next line's row is rejected (its last line
    would also leave the buffer's field, but the check fires first)"""
    assert run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3) < 1e-12
    with pytest.raises(AssertionError, match="writes an element that line"):
        run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3, mutate=_shift_rows("z pass"))


def test_ordering_check_sees_the_buffer(monkeypatch):
    """the happens-before check covers the shared buffer: an overlapped slab schedule whose exchange stream no longer
    waits for the z pass (whose input the x pass overwrites in place) is rejected"""
    def drop_waits(scheds):
        for sc in scheds:
            for st in sc["steps"]:
                if st["stream"] != 0:
                    st["waits"] = []
    assert run_inplace(2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS, 0, 3) < 1e-12
    with pytest.raises(AssertionError, match="without"):
        run_inplace(2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS, 0, 3, mutate=drop_waits)


def test_scale_count_catches_a_second_scale():
    """the replay's count of scalings is not vacuous: a z pass that also applies the scale to what it stores in the
    buffer scales every output value twice"""
    def scale_z(scheds):
        for sc in scheds:
            sc["steps"][0]["scale"] = 3.0
    assert run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3, scale=3.0) < 1e-12
    with pytest.raises(AssertionError, match="scaled 2..2 times"):
        run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3, scale=3.0, mutate=scale_z)
