"""Box-distributed plans (dfft_plan_create_boxes) without a GPU: validation, getters and sizes, byte-identical descriptions
for natural boxes, and numpy replays of every rank's step list (step_replay.py) under the happens-before check, checked
against fftn / rfftn / dctn of the global field on each rank's box.

The replayed cases cover slab, Z_Then_YX and pencil, Peer2Peer and All2All, C2C (with a Bluestein axis), R2C / C2R and DCT,
2x2x2 bricks on 8 ranks, 2x2x1 on 4, z-slabs into an x-slab plan, uneven bricks, out_boxes = in_boxes, bricks of the
Nz/2 + 1 grid, a batch of 2, a scale, partial d in both directions and a kept x axis."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest
import scipy.fft as sf

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import lib

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C, DCT = dfft.C2C, dfft.R2C, dfft.DCT
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
ERR_INVALID, ERR_UNSUPPORTED = -1, -5


# ---- boxes ------------------------------------------------------------------------------------------------------------------
def cuts(n, parts, uneven=False, even=False):
    """part boundaries of an axis of n points: balanced, or with the first part about half as big (uneven); even: every
    boundary even (the real z side of R2C plans)"""
    if uneven:
        w = [1] + [2] * (parts - 1)
        b = [round(n * sum(w[:i]) / sum(w)) for i in range(parts + 1)]
    else:
        b = [i * n // parts for i in range(parts + 1)]
    if even:
        b = [v - v % 2 for v in b]
    assert all(b[i] < b[i + 1] for i in range(parts)), (n, parts, b)
    return b


def bricks(grid, parts, uneven=False, even_z=False):
    """px x py x pz bricks of grid in rank order (x outermost)"""
    cx, cy, cz = (cuts(grid[a], parts[a], uneven, even_z and a == 2) for a in range(3))
    return tuple(((cx[i], cy[j], cz[k]), (cx[i + 1], cy[j + 1], cz[k + 1]))
                 for i in range(parts[0]) for j in range(parts[1]) for k in range(parts[2]))


def natural(p, which):
    """the plan's own layout `which` (0 input, 3 output) of every rank, as boxes"""
    out = []
    for r in range(p.P):
        s, o = (C.c_size_t * 3)(), (C.c_size_t * 3)()
        p1 = p.p1 if p.decomp == PE else p.P  # slab decompositions: the rank count
        assert lib().dfft_layout(p.decomp, p.transform, *p.shape, p1, p.p2, r, which, s, o) == 0
        out.append((tuple(o), tuple(a + b for a, b in zip(o, s))))
    return tuple(out)


def nzc(p):
    return p.shape[2] // 2 + 1 if p.transform == R2C else p.shape[2]


# ---- references -----------------------------------------------------------------------------------------------------------
def transformed(p, d):
    return [a for a in (2, 1, 0)[:d] if p.axes is None or p.axes[a]]


def forward(p, x, d):
    ax = transformed(p, d)
    if p.transform == DCT:
        return sf.dctn(x, type=2, axes=ax) if ax else x.copy()
    if p.transform == R2C:
        X = np.fft.rfft(x, axis=2)
        return np.fft.fftn(X, axes=[a for a in ax if a != 2]) if len(ax) > 1 else X
    return np.fft.fftn(x, axes=ax) if ax else x.copy()


def inverse(p, X, d):
    ax = transformed(p, d)
    if p.transform == DCT:
        return sf.idctn(X, type=2, axes=ax) * np.prod([2 * p.shape[a] for a in ax]) if ax else X.copy()
    n = np.prod([p.shape[a] for a in ax])
    if p.transform == R2C:
        rest = [a for a in ax if a != 2]
        Y = np.fft.ifftn(X, axes=rest) if rest else X
        return np.fft.irfft(Y, n=p.shape[2], axis=2) * n
    return np.fft.ifftn(X, axes=ax) * n if ax else X.copy()


def replay(p, inv, d, seed=0):
    """replays every rank of plan p; returns the worst relative error of the output boxes against the reference"""
    rng = np.random.default_rng(seed)
    real = p.transform in (R2C, DCT)
    xs = [rng.standard_normal(p.shape) + (0 if real else 1j * rng.standard_normal(p.shape)) for _ in range(p.fields)]
    scale = 1.0 if p.scale is None else p.scale[1 if inv else 0]
    if inv:  # the spectrum of a field (R2C: Hermitian), whose inverse is known
        src = [forward(p, x, d) for x in xs]
        want = [inverse(p, X, d) * scale for X in src]
    else:
        src = xs
        want = [forward(p, x, d) * scale for x in xs]
    return R.error(R.replay(p, inv, d, src), want)


def plan(P, decomp, shape, p1=1, p2=1, transform=C2C, in_boxes=None, out_boxes=None, **kw):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, in_boxes=in_boxes, out_boxes=out_boxes, **kw)


# ---- validation -------------------------------------------------------------------------------------------------------------
def rc_of(p, rank=0):
    rc, msg, c, h = R.create(p, rank)
    if rc == 0:
        lib().dfft_plan_destroy(h)
    lib().dfft_comm_destroy(c)
    return rc, msg


def test_validation():
    shape = (8, 8, 16)
    good = bricks(shape, (2, 2, 1))
    assert rc_of(plan(4, SL, shape, in_boxes=good))[0] == 0
    bad = {
        "empty": ((good[0][0], (4, 4, 0)),) + good[1:],
        "outside": (((0, 0, 0), (4, 4, 17)),) + good[1:],
        "overlap": (((0, 0, 0), (4, 5, 16)),) + good[1:],
        "gap": (((0, 0, 0), (4, 3, 16)),) + good[1:],
        "inverted": (((4, 0, 0), (0, 4, 16)),) + good[1:],
    }
    for name, boxes in bad.items():
        rc, msg = rc_of(plan(4, SL, shape, in_boxes=boxes))
        assert rc == ERR_INVALID and "tile" in msg, name
        rc, msg = rc_of(plan(4, SL, shape, out_boxes=boxes))
        assert rc == ERR_INVALID and "tile" in msg, name
    # the output grid of R2C is Nz/2 + 1 deep: the physical grid's bricks do not tile it
    assert rc_of(plan(4, SL, shape, transform=R2C, out_boxes=good))[0] == ERR_INVALID
    assert rc_of(plan(4, SL, shape, transform=R2C, out_boxes=bricks((8, 8, 9), (2, 2, 1))))[0] == 0
    # one rank: the whole grid only
    assert rc_of(plan(1, SL, shape, in_boxes=(((0, 0, 0), shape),)))[0] == 0
    assert rc_of(plan(1, SL, shape, in_boxes=(((0, 0, 0), (8, 8, 8)),)))[0] == ERR_INVALID
    # transforms: C2C, R2C, DCT, DST only (4: R2HC, 16 / 17: DCT-I / DST-I, 19 / 20: type IV)
    for t in (4, 16, 17, 19, 20, 7):
        assert rc_of(plan(4, SL, shape, transform=t, in_boxes=good))[0] == ERR_INVALID, t
    assert rc_of(plan(4, SL, shape, transform=dfft.DST, in_boxes=good))[0] == 0
    # R2C real rows move as pairs: odd z bounds of in_boxes are not supported
    odd = (((0, 0, 0), (8, 8, 7)), ((0, 0, 7), (8, 8, 16)))
    assert rc_of(plan(2, SL, shape, transform=R2C, in_boxes=odd))[0] == ERR_UNSUPPORTED
    assert rc_of(plan(2, SL, shape, transform=C2C, in_boxes=odd))[0] == 0


def test_python_refusals():
    # a geometry-only communicator: each refusal comes before a plan is made
    comm = dfft.Comm.__new__(dfft.Comm)
    comm._h = C.c_void_p()
    assert lib().dfft_comm_create_dry(0, 1, C.byref(comm._h)) == 0
    comm.rank, comm.size, comm.device = 0, 1, 0
    whole = [((0, 0, 0), (8, 8, 8))]
    for kw in ({"inplace": True}, {"spectral": (4, 4, 4)}, {"components": 2}):
        f = dfft.MPIcuFFT_Slab(dfft.Configurations(), comm, transform="c2c")
        with pytest.raises(ValueError):
            f.initFFT(dfft.GlobalSize(8, 8, 8), None, False, in_boxes=whole, **kw)
    f = dfft.MPIcuFFT_Slab(dfft.Configurations(), comm, transform=("dct", "dst", "dct"))
    with pytest.raises(ValueError):
        f.initFFT(dfft.GlobalSize(8, 8, 8), None, False, out_boxes=whole)
    f = dfft.MPIcuFFT_Slab(dfft.Configurations(), comm, transform="c2c")
    with pytest.raises(ValueError):
        f.initFFT(dfft.GlobalSize(8, 8, 8), None, False, in_boxes=whole * 2)
    f.initFFT(dfft.GlobalSize(8, 8, 8), None, False, in_boxes=whole, out_boxes=whole)  # the plain plan
    assert list(f.getInSize()) == [8, 8, 8]
    f.destroy()
    comm.destroy()


# ---- getters and sizes ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("transform", [C2C, R2C, DCT])
def test_getters_and_sizes(transform):
    shape = (8, 12, 16) if transform == C2C else (8, 8, 16)
    p = plan(8, PE, shape, 2, 4, transform=transform)
    ib = bricks(shape, (2, 2, 2), uneven=True, even_z=transform == R2C)
    ob = bricks((8, shape[1], nzc(p)), (2, 1, 4))
    p = plan(8, PE, shape, 2, 4, transform=transform, in_boxes=ib, out_boxes=ob)
    esize = 16 if transform != DCT else 8
    for r in range(p.P):
        sc = R.describe(p, r, 0, 3)
        lay = sc["layouts"]
        (lo, hi) = ib[r]
        assert lay[0] == ([h - l for l, h in zip(lo, hi)], list(lo))
        (lo, hi) = ob[r]
        assert lay[3] == ([h - l for l, h in zip(lo, hi)], list(lo))
        for w in (1, 2):  # the spectral side of partial execs keeps the natural layouts
            s, o = (C.c_size_t * 3)(), (C.c_size_t * 3)()
            assert lib().dfft_layout(PE, transform, *shape, 2, 4, r, w, s, o) == 0
            assert lay[w] == (list(s), list(o))
        vol_in = np.prod(lay[0][0]) * (esize // 2 if transform == R2C else esize)
        vol_out = np.prod(lay[3][0]) * esize
        assert sc["domain_bytes"] >= max(vol_in, vol_out)
        assert sc["work_bytes"] == sc["slot_bytes"] * sc["nslots"]
        assert sc["slot_bytes"] >= max(np.prod(np.subtract(h, l)) for l, h in ob) * esize
        assert sc["in_boxes"] == [list(l) + list(h) for l, h in ib]
        assert sc["out_boxes"] == [list(l) + list(h) for l, h in ob]


# ---- natural boxes make today's plan ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,decomp,shape,p1,p2,send", [
    (1, SL, (512, 512, 512), 1, 1, SYNC),    # the fused z + y stage
    (4, SL, (64, 64, 64), 1, 1, STREAMS),    # the overlapped slab schedule
    (4, PE, (16, 32, 32), 2, 2, SYNC),
    (2, ZY, (16, 16, 32), 1, 1, SYNC),
])
def test_natural_boxes_are_the_plain_plan(P, decomp, shape, p1, p2, send):
    base = plan(P, decomp, shape, p1, p2, send=send, batch=1)
    nat_in, nat_out = natural(base, 0), natural(base, 3)
    variants = [plan(P, decomp, shape, p1, p2, send=send, in_boxes=nat_in, out_boxes=nat_out),
                plan(P, decomp, shape, p1, p2, send=send, in_boxes=nat_in),
                plan(P, decomp, shape, p1, p2, send=send, out_boxes=nat_out)]
    for r in range(P):
        for inv in (0, 1):
            want = R.describe_text(base, r, inv, 3)
            if send == STREAMS:
                assert json.loads(want)["overlapped"]
            if P == 1:
                assert "zy pass" in want or "yz pass" in want
            for v in variants:
                assert R.describe_text(v, r, inv, 3) == want


def test_null_boxes_are_the_plain_plan():
    c, h = C.c_void_p(), C.c_void_p()
    assert lib().dfft_comm_create_dry(0, 4, C.byref(c)) == 0
    cfg = C.byref(dfft._lib.dfft_config(1, 0, P2P, STREAMS, None, P2P, STREAMS))
    assert lib().dfft_plan_create_boxes(c, cfg, SL, dfft.F64, C2C, 64, 64, 64, 1, 1, None, None, 1, 1, C.byref(h)) == 0
    want = R.describe_text(plan(4, SL, (64, 64, 64), send=STREAMS, batch=1), 0, 0, 3)
    assert R.describe_raw(h, 0, 3) == want
    lib().dfft_plan_destroy(h)
    lib().dfft_comm_destroy(c)


def test_boxed_plans_run_the_sequential_schedule():
    shape = (32, 32, 32)
    p = plan(4, SL, shape, send=STREAMS, in_boxes=bricks(shape, (2, 2, 1)))
    for inv in (0, 1):
        sc = R.describe(p, 0, inv, 3)
        assert not sc["overlapped"]
        labels = [s["label"] for s in sc["steps"]]
        assert labels.count("reshape in" if not inv else "reshape out") == 4
        assert "zy pass" not in labels


# ---- replays ----------------------------------------------------------------------------------------------------------------
S3 = (8, 8, 16)
CASES = [
    # (id, P, decomp, shape, p1, p2, transform, in_boxes, out_boxes)
    ("slab-bricks222", 8, SL, S3, 1, 1, C2C, bricks(S3, (2, 2, 2)), bricks(S3, (2, 2, 2))),
    ("slab-bricks221-r2c", 4, SL, S3, 1, 1, R2C, bricks(S3, (2, 2, 1)), bricks((8, 8, 9), (2, 2, 1))),
    ("slab-zslabs-into-xslabs", 4, SL, S3, 1, 1, C2C, bricks(S3, (1, 1, 4)), None),
    ("zyx-bricks221", 4, ZY, S3, 1, 1, C2C, bricks(S3, (2, 2, 1)), bricks(S3, (1, 2, 2))),
    ("zyx-uneven-dct", 4, ZY, S3, 1, 1, DCT, bricks(S3, (2, 1, 2), uneven=True), bricks(S3, (2, 2, 1), uneven=True)),
    ("pencil-bricks222", 8, PE, S3, 2, 4, C2C, bricks(S3, (2, 2, 2)), bricks(S3, (2, 2, 2))),
    ("pencil-uneven-r2c", 4, PE, S3, 2, 2, R2C, bricks(S3, (2, 2, 1), uneven=True, even_z=True), bricks((8, 8, 9), (1, 2, 2), uneven=True)),
    ("pencil-bluestein", 4, PE, (8, 12, 16), 2, 2, C2C, bricks((8, 12, 16), (1, 2, 2), uneven=True), None),
    ("slab-dct-out-only", 4, SL, S3, 1, 1, DCT, None, bricks(S3, (2, 1, 2))),
]
SAME = bricks(S3, (2, 2, 1), uneven=True)
CASES.append(("slab-out-equals-in", 4, SL, S3, 1, 1, C2C, SAME, SAME))


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_replay(case, inv, comm):
    _, P, decomp, shape, p1, p2, transform, ib, ob = case
    p = plan(P, decomp, shape, p1, p2, transform=transform, in_boxes=ib, out_boxes=ob, comm=comm)
    assert replay(p, inv, 3) < 1e-12


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("decomp,p1,p2", [(SL, 1, 1), (ZY, 1, 1), (PE, 2, 2)], ids=["slab", "zyx", "pencil"])
def test_replay_partial(decomp, p1, p2, d, inv, comm):
    """in_boxes apply to the physical side of every d; out_boxes only to d = 3"""
    if decomp == ZY and inv and d == 2:
        pytest.skip("Z_Then_YX offers no partial inverse of d = 2")
    p = plan(4, decomp, S3, p1, p2, transform=C2C, in_boxes=bricks(S3, (2, 2, 1), uneven=True), out_boxes=bricks(S3, (1, 2, 2)), comm=comm)
    assert replay(p, inv, d) < 1e-12


@pytest.mark.parametrize("comm", [P2P, A2A], ids=["p2p", "a2a"])
@pytest.mark.parametrize("transform", [C2C, R2C])
def test_replay_batch_scale(transform, comm):
    ob = bricks((8, 8, nzc(plan(1, SL, S3, transform=transform))), (2, 2, 1))
    p = plan(4, PE, S3, 2, 2, transform=transform, in_boxes=bricks(S3, (2, 1, 2)), out_boxes=ob, comm=comm, batch=2, scale=(0.5, 1 / 96))
    for inv in (0, 1):
        assert replay(p, inv, 3) < 1e-12  # the replay also checks that every output value is scaled exactly once


@pytest.mark.parametrize("inv", [0, 1], ids=["fwd", "inv"])
@pytest.mark.parametrize("decomp,p1,p2", [(SL, 1, 1), (PE, 2, 2)], ids=["slab", "pencil"])
def test_replay_x_kept(decomp, p1, p2, inv):
    p = plan(4, decomp, S3, p1, p2, in_boxes=bricks(S3, (2, 2, 1)), out_boxes=bricks(S3, (1, 2, 2)), axes=(0, 1, 1))
    assert replay(p, inv, 3) < 1e-12


def test_slot_rule_catches_a_missing_reshape_rendezvous():
    p = plan(4, SL, S3, in_boxes=bricks(S3, (2, 2, 1)))

    def drop(scheds):
        for sc in scheds:
            sc["steps"] = [s for s in sc["steps"] if s["label"] != "reshape rendezvous"]
    with pytest.raises(AssertionError):
        R.replay(p, 0, 3, [np.zeros(S3, dtype=complex)], mutate=drop)


def test_slot_rule_refuses_remote_reads_outside_the_output_gathers():
    """the gathers of the output reshape are the only passes that read a peer's slot: relabelled, they fail the replay"""
    p = plan(4, SL, S3, out_boxes=bricks(S3, (1, 2, 2)))

    def relabel(scheds):
        for sc in scheds:
            for s in sc["steps"]:
                if s["label"] == "reshape out":
                    s["label"] = "reshape gather"
    with pytest.raises(AssertionError, match="output gathers"):
        R.replay(p, 0, 3, [np.zeros(S3, dtype=complex)], mutate=relabel)
