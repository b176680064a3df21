"""Plans with strides (dfft_plan_set_strides) without a GPU: refusals, getters, descriptions, the schedule they run, and numpy
replays of every rank's step list (step_replay.py) under the happens-before check, on caller arrays whose ghost layers
hold a poison that no pass may read or overwrite.

Each replay is checked against the same plan without strides, replayed the same way on dense arrays (the step lists of
those are checked against numpy references by the other replay tests).  The cases cover slab, Z_Then_YX and pencil with
Peer2Peer and All2All, uneven splits and the blocked hand-over with leftover columns; C2C with a Bluestein axis, R2C / C2R,
DCT and a mixed (r2hc, dct1, dst4) plan; a batch of 2 with a gap between fields, a scale; partial d both ways, a kept x axis,
a padded plan and a box plan."""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import replace

import numpy as np
import pytest
import scipy.fft as sf

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import lib
from test_boxes import bricks

R.R2R.setdefault("dct4", lambda x, inv: sf.dct(x, type=4, axis=2))
R.R2R.setdefault("dst4", lambda x, inv: sf.dst(x, type=4, axis=2))

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C, DCT, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.R2HC
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
ERR_INVALID, ERR_STATE, ERR_UNSUPPORTED = -1, -4, -5


def plan(P, decomp, shape, p1=1, p2=1, embed="both", **kw):
    return R.Plan(P, decomp, tuple(shape), p1, p2, embed=embed, **kw)


def dense(p):
    """the same plan without strides"""
    return replace(p, embed=None)


# ---- refusals, getters, descriptions ----------------------------------------------------------------------------------------
def make(p, rank=0):
    """rank's plan of p before any setter"""
    rc, msg, c, h = R.create(dense(p), rank)
    assert rc == 0, msg
    return c, h


def close(c, h):
    lib().dfft_plan_destroy(h)
    lib().dfft_comm_destroy(c)


def set_strides(h, i, o):
    arr = lambda s: None if s is None else (C.c_longlong * 3)(*s)
    rc = lib().dfft_plan_set_strides(h, arr(i), arr(o))
    return rc, (lib().dfft_last_error_string() or b"").decode()


def test_validation():
    c, h = make(plan(2, SL, (8, 6, 10)))  # rank 0: in [4][6][10], out [8][3][10]
    try:
        assert set_strides(h, (4 * 6 * 10, 6 * 10, 10), (8 * 3 * 10, 3 * 10, 10))[0] == 0  # dense strides are valid
        for bad in [(400, 60, 9), (400, 59, 10), (239, 60, 10), (0, 0, 0), (-1, 60, 10)]:
            rc, msg = set_strides(h, bad, None)
            assert rc == ERR_INVALID and "in_strides" in msg, (bad, msg)
        rc, msg = set_strides(h, None, (8 * 36, 36, 11 - 2))
        assert rc == ERR_INVALID and "out_strides" in msg
        assert set_strides(h, (1000, 100, 12), (1000, 40, 12))[0] == 0
    finally:
        close(c, h)
    # the real side of R2C / C2R moves pairs of reals: even strides only; its output side takes any
    c, h = make(plan(1, SL, (4, 4, 8), transform=R2C))
    try:
        for bad in [(500, 100, 11), (500, 101, 12), (501, 100, 12)]:
            rc, msg = set_strides(h, bad, None)
            assert rc == ERR_INVALID and "even" in msg, bad
        assert set_strides(h, (500, 100, 12), (301, 75, 5))[0] == 0
    finally:
        close(c, h)


@pytest.mark.parametrize("kw,word", [({"inplace": True}, "in-place"), ({"components": 2}, "interleaved")])
def test_refusals(kw, word):
    c, h = make(plan(1, SL, (8, 8, 8), **kw))
    try:
        rc, msg = set_strides(h, (1000, 100, 10), None)
        assert rc == ERR_UNSUPPORTED and word in msg, msg
    finally:
        close(c, h)


def test_state_after_the_schedule_is_built():
    c, h = make(plan(1, SL, (8, 8, 8)))
    try:
        R.describe_raw(h, 0, 3)
        rc, msg = set_strides(h, (1000, 100, 10), None)
        assert rc == ERR_STATE and "before the first exec" in msg
    finally:
        close(c, h)


def test_getters_and_describe():
    c, h = make(plan(4, PE, (8, 8, 16), 2, 2, transform=R2C))
    try:
        i, o = (C.c_longlong * 3)(), (C.c_longlong * 3)()
        assert lib().dfft_plan_get_strides(h, i, o) == 0
        # rank 0: in [4][4][16] reals, out [8][4][5] complex; without strides the dense ones
        assert tuple(i) == (4 * 4 * 16, 4 * 16, 16) and tuple(o) == (8 * 4 * 5, 4 * 5, 5)
        assert set_strides(h, (2000, 200, 20), None)[0] == 0
        assert lib().dfft_plan_get_strides(h, i, None) == 0 and tuple(i) == (2000, 200, 20)
        assert lib().dfft_plan_get_strides(h, None, o) == 0 and tuple(o) == (8 * 4 * 5, 4 * 5, 5)
        sc = json.loads(R.describe_raw(h, 0, 3))
        assert sc["in_strides"] == [2000, 200, 20] and "out_strides" not in sc
    finally:
        close(c, h)
    sc = R.describe(plan(2, ZY, (8, 8, 8), embed="both", halo=1, batch=2, gap=3), 1, 1, 3)
    assert sc["in_strides"] == list(R.strides([4, 8, 8], 1, 3)) and sc["out_strides"] == list(R.strides([8, 8, 4], 1, 3))
    assert sc["field_in"] == sc["out_strides"][0] * 16 and sc["field_out"] == sc["in_strides"][0] * 16


@pytest.mark.parametrize("P,decomp,shape,send,batch,label", [
    (1, SL, (512, 512, 512), SYNC, None, "zy pass"),     # the fused z + y stage
    (4, SL, (64, 64, 64), STREAMS, None, None),          # the overlapped slab schedule
    (1, SL, (32, 32, 32), SYNC, 4, "batched pass"),      # the one-launch batched stage
])
def test_plans_without_strides_keep_their_schedule(P, decomp, shape, send, batch, label):
    """null strides describe byte for byte as the plan that never called the setter; strides take the sequential schedule"""
    base = plan(P, decomp, shape, send=send, batch=batch, embed="")
    for r in range(P):
        for inv in (0, 1):
            want = R.describe_text(base, r, inv, 3)
            assert "in_strides" not in want and "out_strides" not in want
            if label:
                assert label in want or label.replace("zy", "yz") in want
            else:
                assert json.loads(want)["overlapped"]
            c, h = make(base, r)
            try:
                assert set_strides(h, None, None)[0] == 0
                assert R.describe_raw(h, inv, 3) == want
            finally:
                close(c, h)
            got = R.describe(plan(P, decomp, shape, send=send, batch=batch, halo=1), r, inv, 3)
            assert not got["overlapped"]
            labels = [s["label"] for s in got["steps"]]
            assert not any(l.startswith(("zy pass", "yz pass", "batched pass")) for l in labels), labels


# ---- replays ----------------------------------------------------------------------------------------------------------------
def inputs(p, inv, d, seed=0):
    """a global input per field for direction inv: the physical grid, or the forward transform's output (the spectrum of
    the same plan without strides, so that R2C inverses get Hermitian input)"""
    rng = np.random.default_rng(seed)
    real = p.transform in (R2C, DCT) or p.kinds is not None
    xs = [rng.standard_normal(p.shape) + (0 if real else 1j * rng.standard_normal(p.shape)) for _ in range(p.fields)]
    if not inv:
        return xs
    return R.assemble(R.replay(dense(p), 0, d, xs))


def check(p, inv, d=3):
    x = inputs(p, inv, d)
    want = R.assemble(R.replay(dense(p), inv, d, x))
    got = R.replay(p, inv, d, x)
    assert R.error(got, want) < 1e-14


S = (8, 12, 16)
KINDS = (R2HC, dfft.DCT1, dfft.DST4)
CASES = [
    # (id, P, decomp, shape, p1, p2, kw)
    ("slab-1", 1, SL, S, 1, 1, {}),
    ("slab-3-uneven", 3, SL, (8, 8, 16), 1, 1, {}),
    ("zyx-1", 1, ZY, S, 1, 1, {}),
    ("zyx-3-uneven", 3, ZY, (8, 8, 16), 1, 1, {}),
    ("pencil-1", 1, PE, S, 1, 1, {}),
    ("pencil-2x2", 4, PE, S, 2, 2, {}),
    ("pencil-2x3-uneven", 6, PE, (8, 8, 16), 2, 3, {}),
    ("pencil-2x3-bluestein", 6, PE, (7, 10, 11), 2, 3, {}),
    ("pencil-2x4", 8, PE, (8, 8, 8), 2, 4, {}),
    ("slab-bluestein", 2, SL, (6, 12, 10), 1, 1, {}),
    ("pencil-r2c", 4, PE, (8, 8, 16), 2, 2, {"transform": R2C}),
    ("zyx-r2c", 3, ZY, (8, 8, 16), 1, 1, {"transform": R2C}),
    ("slab-dct", 3, SL, (8, 8, 16), 1, 1, {"transform": DCT}),
    ("pencil-mixed", 4, PE, (8, 9, 8), 2, 2, {"transform": R2HC, "kinds": KINDS}),
    ("slab-mixed", 1, SL, (8, 9, 8), 1, 1, {"transform": R2HC, "kinds": KINDS}),
]


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_replay(case, inv, comm):
    _, P, decomp, shape, p1, p2, kw = case
    check(plan(P, decomp, shape, p1, p2, comm=comm, **kw), inv)


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("decomp,P,p1,p2,nz", [(SL, 3, 1, 1, 18), (PE, 4, 2, 2, 36), (SL, 1, 1, 1, 18)], ids=["slab", "pencil", "slab-1"])
def test_replay_blocked_tails(decomp, P, p1, p2, nz, inv, comm, monkeypatch):
    """the blocked hand-over with leftover columns (4-column blocks, 18 z columns per rank): its tail passes"""
    monkeypatch.setenv("DFFT_BLOCKED", "4")
    p = plan(P, decomp, (8, 8, nz), p1, p2, comm=comm)
    if comm == P2P:
        labels = [s["label"] for s in R.describe(p, 0, inv, 3)["steps"]]
        assert "x pass (tail)" in labels or "y pass (tail)" in labels, labels
    check(p, inv)


@pytest.mark.parametrize("embed", ["in", "out", "both"])
@pytest.mark.parametrize("transform", [C2C, R2C])
def test_replay_batch_gap_scale(transform, embed):
    """batch 2, fields further apart than the blocks, one side or both with strides, a scale (each output value scaled once)"""
    p = plan(4, PE, (8, 8, 16), 2, 2, transform=transform, batch=2, gap=6, embed=embed, scale=(0.5, 1 / 96))
    for inv in (0, 1):
        check(p, inv)


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("decomp,p1,p2", [(SL, 1, 1), (ZY, 1, 1), (PE, 2, 2)], ids=["slab", "zyx", "pencil"])
def test_replay_partial(decomp, p1, p2, d, inv, comm):
    """in_strides apply to the physical side of every d; the spectral side of partial execs stays dense"""
    if decomp == ZY and inv and d == 2:
        pytest.skip("Z_Then_YX offers no partial inverse of d = 2")
    p = plan(4, decomp, S, p1, p2, comm=comm)
    sc = R.describe(p, 0, inv, d)
    assert "in_strides" in sc and "out_strides" in sc
    check(p, inv, d)


@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("decomp,P,p1,p2", [(SL, 4, 1, 1), (PE, 4, 2, 2), (SL, 1, 1, 1)], ids=["slab", "pencil", "slab-1"])
def test_replay_x_kept(decomp, P, p1, p2, inv):
    check(plan(P, decomp, S, p1, p2, axes=(0, 1, 1)), inv)


@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("transform", [C2C, R2C])
def test_replay_padded(transform, inv):
    check(plan(4, PE, (8, 8, 16), 2, 2, transform=transform, spectral=(6, 4, 10)), inv)


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
def test_replay_boxes(inv, comm):
    """the box is the embedded block: the reshape copies read and write the caller's arrays through the strides"""
    p = plan(4, SL, (8, 8, 16), comm=comm, in_boxes=bricks((8, 8, 16), (2, 2, 1), uneven=True), out_boxes=bricks((8, 8, 16), (1, 2, 2)))
    check(p, inv)


def test_ghost_rule_catches_a_view_off_its_block():
    """a pass view moved by one element reaches into the ghost layers: the replay refuses it"""
    p = plan(1, SL, S)

    def shift(scheds):
        for sc in scheds:
            st = next(s for s in sc["steps"] if s["type"] == 0 and s["in_user"] == 1)
            st["in"]["segs"][0]["base"] -= sc["esize"]
    with pytest.raises(AssertionError, match="ghost"):
        R.replay(p, 0, 3, inputs(p, 0, 3), mutate=shift)
