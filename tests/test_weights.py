"""Per-axis spectral weights (dfft_plan_set_weights) without a GPU: refusals and the state rule, the describe keys, and
numpy replays of every rank's weighted step list against W * fftn(x) and ifftn(W * X).

A weighted pass ("weighted", "axis") multiplies its spectral side by the weights of its axis: forward the values it stores,
inverse the values it loads.  weights_replay.py runs the step lists through step_replay's engine with numpy tables applied
the same way, so a pass that applied no weight, the wrong axis's, or the weight at the wrong index (the stored K positions
of padded plans) shows up against the reference."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
import weights_replay as WR
from distributedfft_b200._lib import lib
from step_replay import positions

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C = dfft.C2C, dfft.R2C
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
OK, ERR_INVALID, ERR_STATE, ERR_UNSUPPORTED = 0, -1, -4, -5


def err():
    return (lib().dfft_last_error_string() or b"").decode()


def ptrs(*vals):
    return (C.c_void_p * 3)(*vals)


# ---- references -----------------------------------------------------------------------------------------------------------
def spectral_len(p, a):
    k = (p.spectral or p.shape)[a]
    return k // 2 + 1 if p.transform == R2C and a == 2 else k


def random_weights(p, seed, which=(0, 1, 2)):
    rng = np.random.default_rng(seed)
    return tuple(rng.standard_normal(spectral_len(p, a)) + 1j * rng.standard_normal(spectral_len(p, a)) if a in which else None
                 for a in range(3))


def along(w, axis):
    shape = [1, 1, 1]
    shape[axis] = w.size
    return w.reshape(shape)


def transformed(p, d):
    return [a for a in (2, 1, 0)[:d] if p.axes is None or p.axes[a]]


def fwd_ref(p, ws, x, d):
    """the first d axes (z, y, x order) of the data block zero-embedded to N, transformed, truncated to K, times the weights"""
    spec = p.spectral or p.shape
    for axis in transformed(p, d):
        half = p.transform == R2C and axis == 2
        pad = [(0, 0)] * 3
        pad[axis] = (0, p.shape[axis] - x.shape[axis])
        x = np.pad(x, pad)
        x = np.fft.rfft(x, axis=2) if half else np.fft.fft(x, axis=axis)
        x = np.take(x, positions(p.shape[axis], spec[axis], half), axis=axis)
        if ws[axis] is not None:
            x = x * along(ws[axis], axis)
    return x


def inv_ref(p, ws, X, d):
    """the unnormalised inverse of the weighted, zero-embedded spectrum along the first d axes, truncated to the data block"""
    spec, data = p.spectral or p.shape, p.data or p.shape
    for axis in (0, 1, 2):
        if axis not in transformed(p, d):
            continue
        if ws[axis] is not None:
            X = X * along(ws[axis], axis)
        half = p.transform == R2C and axis == 2
        n = p.shape[axis]
        full = list(X.shape)
        full[axis] = n // 2 + 1 if half else n
        E = np.zeros(full, dtype=np.result_type(X.dtype, np.complex128))  # long double stays long double
        idx = [slice(None)] * 3
        idx[axis] = positions(n, spec[axis], half)
        E[tuple(idx)] = X
        X = np.fft.irfft(E, n=n, axis=2) * n if half else np.fft.ifft(E, axis=axis) * n
        X = np.take(X, np.arange(data[axis]), axis=axis)
    return X


def replay(pw, inverse, d, seed=0):
    """replays every rank of the weighted plan pw = (plan, tables); returns the worst rel-L2 error of any output block
    against the reference"""
    p, ws = pw
    scheds = [WR.describe(p, ws, r, inverse, d) for r in range(p.P)]
    assert not scheds[0]["overlapped"]
    assert scheds[0]["weights"] == [int(w is not None) for w in ws]
    rng = np.random.default_rng(seed + 3 * d + inverse)
    block = p.data or p.shape
    xs = [rng.standard_normal(block) + (0 if p.transform == R2C else 1j * rng.standard_normal(block)) for _ in range(p.fields)]
    scale = 1.0 if p.scale is None else p.scale[1 if inverse else 0]
    if inverse:  # the unweighted spectrum of a field (R2C: Hermitian)
        src = [fwd_ref(p, (None, None, None), x, d) for x in xs]
        want = [inv_ref(p, ws, X, d) * scale for X in src]
    else:
        src, want = xs, [fwd_ref(p, ws, x, d) * scale for x in xs]
    return R.error(WR.replay(p, ws, inverse, d, src, scheds), want)


def weighted(P, decomp, shape, p1=1, p2=1, transform=C2C, seed=1, which=(0, 1, 2), **kw):
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, **kw)
    return p, random_weights(p, seed, which)


# ---- refusals and state -----------------------------------------------------------------------------------------------------
def dry(p, rank=0):
    rc, msg, c, plan = R.create(p, rank)
    assert rc == 0, msg
    return c, plan


def close(c, plan):
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


def test_refusals():
    assert lib().dfft_plan_set_weights(None, ptrs(None, None, None)) == ERR_INVALID and "null plan" in err()
    assert lib().dfft_plan_get_weights(None, ptrs(None, None, None)) == ERR_INVALID
    c, plan = dry(R.Plan(1, SL, (8, 8, 8)))
    assert lib().dfft_plan_set_weights(plan, None) == ERR_INVALID and "null plan / weights" in err()
    assert lib().dfft_plan_get_weights(plan, None) == ERR_INVALID
    assert lib().dfft_plan_set_weights(plan, ptrs(None, 4104, None)) == ERR_INVALID and "weights[1] must be aligned to its 16-byte element" in err()
    close(c, plan)
    c, plan = dry(R.Plan(1, SL, (8, 8, 8), prec=dfft.F32))
    assert lib().dfft_plan_set_weights(plan, ptrs(4100, None, None)) == ERR_INVALID and "8-byte element" in err()
    assert lib().dfft_plan_set_weights(plan, ptrs(4104, None, None)) == OK
    close(c, plan)
    for p, msg in ((R.Plan(1, SL, (8, 8, 8), components=2), "interleaved plans of more than one component"),
                   (R.Plan(1, SL, (8, 8, 8), transform=dfft.DCT, kinds=(dfft.DCT,) * 3), "real-to-real plans"),
                   (R.Plan(1, SL, (8, 8, 8), kinds=(dfft.DCT, dfft.R2HC, dfft.R2HC)), "real-to-real plans"),
                   (R.Plan(1, SL, (8, 8, 8), prec=dfft.F16), "spectral weights have no 16-bit storage"),
                   (R.Plan(1, SL, (8, 8, 8), transform=R2C, prec=dfft.BF16), "spectral weights have no 16-bit storage")):
        c, plan = dry(p)
        assert lib().dfft_plan_set_weights(plan, ptrs(None, None, None)) == ERR_UNSUPPORTED and msg in err(), err()
        close(c, plan)
    # one component is an ordinary plan
    c, plan = dry(R.Plan(1, SL, (8, 8, 8), components=1))
    assert lib().dfft_plan_set_weights(plan, ptrs(None, None, None)) == OK
    close(c, plan)


def test_state_rule_and_getter():
    c, plan = dry(R.Plan(2, SL, (8, 8, 16), 2))
    got = ptrs(1, 2, 3)
    assert lib().dfft_plan_get_weights(plan, got) == OK and list(got) == [None, None, None]
    R.describe_raw(plan, 0, 3)
    assert lib().dfft_plan_set_weights(plan, ptrs(16, 32, 48)) == ERR_STATE and "before the first exec" in err()
    close(c, plan)
    c, plan = dry(R.Plan(2, SL, (8, 8, 16), 2))
    assert lib().dfft_plan_set_weights(plan, ptrs(None, None, None)) == OK  # all NULL: a weighted plan all the same
    text = R.describe_raw(plan, 0, 3)
    assert json.loads(text)["weights"] == [0, 0, 0]
    for w in ((16, None, 64), (None, 32, None), (None, None, None)):  # re-pointing after the schedule is built
        assert lib().dfft_plan_set_weights(plan, ptrs(*w)) == OK
        assert lib().dfft_plan_get_weights(plan, got) == OK and list(got) == list(w)
        sc = json.loads(R.describe_raw(plan, 0, 3))
        assert sc["weights"] == [int(v is not None) for v in w]
        # the step list does not depend on which pointers are set
        assert sc["steps"] == json.loads(text)["steps"]
    close(c, plan)


@pytest.mark.parametrize("P,decomp,shape,p1,p2,transform", [
    (1, SL, (8, 16, 32), 1, 1, C2C), (4, SL, (16, 8, 64), 4, 1, R2C), (4, ZY, (8, 8, 16), 4, 1, C2C), (8, PE, (8, 16, 32), 2, 4, R2C)])
def test_describe_keys(P, decomp, shape, p1, p2, transform):
    """weighted plans: the plan-level "weights" and "weighted" / "axis" on each FFT pass; otherwise the plain description"""
    p = R.Plan(P, decomp, shape, p1, p2, transform=transform)
    for inverse in (0, 1):
        for d in (1, 3):
            plain = R.describe(p, 0, inverse, d)
            assert "weights" not in plain and not any("weighted" in st for st in plain["steps"])
            w = WR.describe(p, random_weights(p, 0, (0, 2)), 0, inverse, d)
            assert w["weights"] == [1, 0, 1]
            passes = [st for st in w["steps"] if st["type"] == 0]
            assert passes and all(st["weighted"] == 1 for st in passes)
            assert {st["axis"] for st in passes} == set((2, 1, 0)[:d])
            stripped = {**w, "steps": [{k: v for k, v in st.items() if k not in ("weighted", "axis")} for st in w["steps"]]}
            stripped.pop("weights")
            if P > 1 or d < 3:  # one-rank slab plans of d = 3 may run other stages unweighted
                assert stripped == plain


def test_weighted_plans_run_the_sequential_schedule():
    """the fused z + y stage, the batched stage and the overlapped schedules have no weighted twins"""
    for p, plain_labels in ((R.Plan(1, SL, (512, 256, 256)), "zy pass: z phase"),):
        assert any(st["label"] == plain_labels for st in R.describe(p, 0, 0, 3)["steps"])
        w = WR.describe(p, random_weights(p, 0), 0, 0, 3)
        assert [st["label"] for st in w["steps"] if st["type"] == 0] == ["z pass", "y pass", "x pass"]
    b = R.Plan(1, SL, (32, 32, 32), batch=3)
    assert R.describe(b, 0, 0, 3)["steps"][0]["label"].startswith("batched pass")
    assert all("batched" not in st["label"] for st in WR.describe(b, random_weights(b, 0), 0, 0, 3)["steps"])
    o = R.Plan(8, SL, (32, 16, 256), 8, send=STREAMS)
    assert R.describe(o, 0, 0, 3)["overlapped"]
    assert not WR.describe(o, random_weights(o, 0), 0, 0, 3)["overlapped"]


# ---- replays --------------------------------------------------------------------------------------------------------------------
CASES = [
    # P, decomp, shape, p1, p2, transform, comm
    (1, SL, (8, 16, 32), 1, 1, C2C, P2P),
    (1, SL, (4, 8, 64), 1, 1, R2C, P2P),
    (2, SL, (8, 8, 16), 2, 1, C2C, A2A),
    (3, SL, (8, 16, 16), 3, 1, R2C, P2P),       # uneven split
    (4, SL, (8, 16, 128), 4, 1, R2C, P2P),      # blocked + tail column
    (8, SL, (16, 16, 64), 8, 1, C2C, A2A),
    (1, ZY, (8, 8, 16), 1, 1, C2C, P2P),
    (4, ZY, (8, 4, 32), 4, 1, R2C, P2P),
    (6, ZY, (12, 8, 16), 6, 1, C2C, A2A),
    (1, PE, (8, 8, 16), 1, 1, R2C, P2P),
    (6, PE, (12, 8, 16), 3, 2, C2C, P2P),
    (8, PE, (8, 16, 32), 2, 4, R2C, A2A),
]


@pytest.mark.parametrize("P,decomp,shape,p1,p2,transform,comm", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_replay(P, decomp, shape, p1, p2, transform, comm, inverse):
    assert replay(weighted(P, decomp, shape, p1, p2, transform, comm=comm, seed=P), inverse, 3) < 1e-12


@pytest.mark.parametrize("P,decomp,shape,p1,p2", [(1, SL, (6, 12, 10), 1, 1), (3, SL, (9, 6, 20), 3, 1), (4, ZY, (12, 10, 6), 4, 1),
                                                  (4, PE, (5, 12, 9), 2, 2)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_replay_bluestein(P, decomp, shape, p1, p2, inverse):
    assert replay(weighted(P, decomp, shape, p1, p2), inverse, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("transform", [C2C, R2C])
def test_replay_partial(d, inverse, transform):
    """partial d: the weights of the first d axes apply"""
    assert replay(weighted(8, PE, (8, 16, 32), 2, 4, transform), inverse, d) < 1e-12
    assert replay(weighted(4, SL, (8, 8, 16), 4, 1, transform, comm=A2A), inverse, d) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_replay_batch_scale_and_missing_axes(inverse):
    """batches (the same weights for every field) with a scale; axes without weights"""
    assert replay(weighted(4, PE, (8, 8, 16), 2, 2, R2C, batch=2, scale=(0.5, 1 / 96)), inverse, 3) < 1e-12
    assert replay(weighted(3, SL, (8, 16, 16), 3, 1, C2C, batch=2, scale=(3.0, 0.25), which=(1,)), inverse, 3) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_replay_inplace(inverse):
    assert replay(weighted(4, PE, (8, 8, 16), 2, 2, R2C, inplace=True), inverse, 3) < 1e-12
    assert replay(weighted(1, SL, (8, 16, 32), 1, 1, C2C, inplace=True), inverse, 3) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_replay_kept_axis(inverse):
    """a kept axis ignores its weight; its copy pass is not weighted"""
    for axes in ((0, 1, 1), (1, 0, 1), (1, 1, 0)):
        assert replay(weighted(4, PE, (8, 8, 16), 2, 2, axes=axes), inverse, 3) < 1e-12
    assert replay(weighted(4, SL, (8, 8, 32), 4, 1, R2C, axes=(0, 1, 1)), inverse, 3) < 1e-12


@pytest.mark.parametrize("transform", [C2C, R2C])
@pytest.mark.parametrize("inverse", [0, 1])
def test_replay_padded_and_pruned(transform, inverse):
    """the weights index the K stored positions"""
    assert replay(weighted(4, PE, (8, 16, 32), 2, 2, transform, spectral=(5, 11, 21)), inverse, 3) < 1e-12
    assert replay(weighted(3, SL, (16, 8, 16), 3, 1, transform, spectral=(7, 8, 10)), inverse, 3) < 1e-12
    assert replay(weighted(4, ZY, (8, 16, 16), 4, 1, transform, data=(5, 9, 10)), inverse, 3) < 1e-12
    assert replay(weighted(4, PE, (16, 8, 32), 2, 2, transform, data=(8, 5, 18), spectral=(11, 8, 21)), inverse, 3) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_replay_boxes_and_strides(inverse):
    from test_boxes import bricks
    g = (8, 12, 16)
    p = R.Plan(4, PE, g, 2, 2, in_boxes=bricks(g, (1, 2, 2), uneven=True), out_boxes=bricks(g, (2, 2, 1)))
    assert replay((p, random_weights(p, 5)), inverse, 3) < 1e-12
    assert replay(weighted(4, SL, (8, 8, 16), 4, 1, R2C, embed="both", batch=2, gap=6), inverse, 3) < 1e-12
    assert replay(weighted(2, ZY, (8, 8, 16), 2, 1, C2C, embed="in", halo=1), inverse, 3) < 1e-12
