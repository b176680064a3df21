"""Natural-order distributed 1D transforms (dfft_plan_create_1d_natural) without a GPU: refusals, the default factors, the
getters, describe keys, the unchanged description of dfft_plan_create_1d plans, and replays of every rank's step list on
geometry-only communicators.  Each rank's forward output is compared with its contiguous slice of numpy.fft.fft of the
signal, with no index map."""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np
import pytest

import fft1d_natural_replay as N
import fft1d_replay as F
import step_replay as R
import distributedfft_b200 as dfft
from distributedfft_b200._lib import check, lib

SLAB = dfft.SLAB_ZY_THEN_X
ERR_INVALID, ERR_UNSUPPORTED = -1, -5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fft1d_scrambled_describe.json")


def rng_signal(shape, seed=0):
    g = np.random.default_rng(seed)
    return g.standard_normal(shape) + 1j * g.standard_normal(shape)


def create_rc(P, n, factors=None, prec=dfft.F64, rank=0):
    rc, msg, c, plan = N.create(R.Plan(P, SLAB, (0, 0, 0), prec=prec), n, factors, rank)
    if rc == 0:
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return rc, msg


@pytest.mark.parametrize("P, n, factors, prec, code, text", [
    (1, 1 << 10, None, dfft.F16, ERR_UNSUPPORTED, "1D plans have no 16-bit storage"),
    (1, 1 << 10, None, dfft.BF16, ERR_UNSUPPORTED, "1D plans have no 16-bit storage"),
    (1, 1000, None, dfft.F64, ERR_UNSUPPORTED, "power of two in [8, 2^39]"),
    (1, 1 << 40, None, dfft.F64, ERR_UNSUPPORTED, "power of two in [8, 2^39]"),
    (1, 1 << 15, (6, 64, 64), dfft.F64, ERR_UNSUPPORTED, "powers of two in [2, 8192]"),
    (1, 1 << 15, (32, 32, 16), dfft.F64, ERR_INVALID, "multiply to n"),
    (4, 1 << 12, (2, 64, 32), dfft.F64, ERR_INVALID, "N1 and N2 of a 1D plan must be at least the rank count"),
    (4, 1 << 12, (64, 32, 2), dfft.F64, ERR_INVALID, "N3 of a natural-order 1D plan must be at least the rank count"),
    (3, 1 << 9, (64, 4, 2), dfft.F64, ERR_INVALID, "N3 of a natural-order 1D plan"),
    (16, 1 << 10, None, dfft.F64, ERR_UNSUPPORTED, "with N1, N2 and N3 at least the rank count"),
    (1, 1 << 10, None, 9, ERR_INVALID, "bad precision"),
])
def test_create_refusals(P, n, factors, prec, code, text):
    rc, msg = create_rc(P, n, factors, prec)
    assert rc == code and text in msg, (rc, msg)


def test_scrambled_plan_takes_a_small_n3():
    """the N3 rule is natural order's own: dfft_plan_create_1d still takes N3 below the rank count"""
    rc, msg, c, plan = F.create(R.Plan(4, SLAB, (0, 0, 0)), 1 << 12, (64, 32, 2), 0)
    assert rc == 0, msg
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


def expected_factors(n, P):
    """the factor rule of dfft.h with N3 >= P as well, or None where no split exists"""
    L, lp = n.bit_length() - 1, max(1, (P - 1).bit_length())
    cands = [(l1, l2, L - l1 - l2) for l1 in range(lp, 14) for l2 in range(lp, 14) if lp <= L - l1 - l2 <= 13]
    if not cands:
        return None
    l1, l2, l3 = min(cands, key=lambda c: (max(c) - min(c), -c[0], -c[1]))
    return 1 << l1, 1 << l2, 1 << l3


@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 6, 7, 8])
def test_default_factors(P):
    for L in range(3, 40):
        n = 1 << L
        rc, msg, c, plan = N.create(R.Plan(P, SLAB, (0, 0, 0)), n, None, 0)
        if rc:
            assert rc == ERR_UNSUPPORTED and expected_factors(n, P) is None, (L, P, msg)
            lib().dfft_comm_destroy(c)
            continue
        f = F.factors_of(plan)
        assert f == expected_factors(n, P) and f[0] * f[1] * f[2] == n and min(f) >= P, (L, P, f)
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)


def _triple(fn, plan, *args):
    v = (C.c_size_t * 3)()
    check(fn(plan, *args, v))
    return [int(x) for x in v]


@pytest.mark.parametrize("P", [1, 2, 3, 4, 5, 6, 7, 8])
def test_getters_tile_the_spectrum(P):
    """rank by rank, the out chunks [oz_r][N2][N1] cover [0, n) in order; in chunks are the x-slabs of dfft_plan_create_1d"""
    n = 1 << 15
    shape = N.plan_of(P, n).shape
    n1, n2, n3 = shape
    p = R.Plan(P, SLAB, shape)
    k = 0
    with N.dry_plans(p, n) as plans, F.dry_plans(p, n) as scrambled:
        for r, (plan, ref) in enumerate(zip(plans, scrambled)):
            size, start = _triple(lib().dfft_get_out_size, plan), _triple(lib().dfft_get_out_start, plan)
            assert size[1:] == [n2, n1] and start[1:] == [0, 0], (r, size, start)
            assert start[0] * n1 * n2 == k, (r, start, k)
            k += size[0] * n1 * n2
            assert _triple(lib().dfft_get_partial_size, plan, 3) == size and _triple(lib().dfft_get_partial_start, plan, 3) == start
            assert size[0] in (n3 // P, n3 // P + 1)
            for get in (lib().dfft_get_in_size, lib().dfft_get_in_start):
                assert _triple(get, plan) == _triple(get, ref)
            es = 16
            dom = lib().dfft_get_domain_size(plan)
            assert dom >= es * max(int(np.prod(_triple(lib().dfft_get_in_size, plan))), int(np.prod(size)))
            assert lib().dfft_get_work_size_device(plan) >= lib().dfft_get_work_size_device(ref)
            assert F.factors_of(plan) == shape
    assert k == n


def test_setter_and_exec_refusals():
    rc, msg, c, plan = N.create(R.Plan(1, SLAB, (0, 0, 0)), 1 << 12, None, 0)
    assert rc == 0, msg
    try:
        assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == ERR_UNSUPPORTED
        assert "1D plans transform every axis" in lib().dfft_last_error_string().decode()
        assert lib().dfft_plan_set_strides(plan, (C.c_longlong * 3)(4096, 256, 16), None) == ERR_UNSUPPORTED
        assert lib().dfft_plan_set_weights(plan, (C.c_void_p * 3)(None, None, 1 << 40)) == ERR_UNSUPPORTED
        assert "1D plans have no spectral weights" in lib().dfft_last_error_string().decode()
        for d in (1, 2):
            need = C.c_size_t()
            assert lib().dfft_plan_describe(plan, 0, d, None, 0, C.byref(need)) == ERR_UNSUPPORTED
            assert "d = 3" in lib().dfft_last_error_string().decode()
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)


def test_python_binding_refusals():
    """the binding takes natural=True with signal only, and refuses it elsewhere before it creates a plan"""
    def binding(cls, transform):
        p = cls.__new__(cls)
        p.config, p.precision, p.kinds, p.transform = dfft.Configurations(), dfft.F64, None, transform
        p.comm = type("DryComm", (), {"size": 1, "_h": None})()
        return p

    slab = binding(dfft.MPIcuFFT_Slab, dfft.C2C)
    with pytest.raises(ValueError, match="natural belongs to a 1D plan"):
        slab.initFFT(dfft.GlobalSize(16, 16, 16), natural=True)
    with pytest.raises(ValueError, match="1D plans are C2C"):
        slab.initFFT(None, signal=1 << 12, natural=True, batch=2)
    for kw in ({"inplace": True}, {"spectral": (4, 4, 4)}, {"components": 2}):
        with pytest.raises(ValueError, match="1D plans are out of place"):
            slab.initFFT(None, signal=1 << 12, natural=True, **kw)


@pytest.mark.parametrize("P, comm", [(1, 0), (3, 0), (3, 1), (4, 0)])
def test_describe_keys(P, comm):
    n, shape = 1 << 12, (16, 16, 16)
    p = N.plan_of(P, n, shape, comm=comm)
    for inverse in (0, 1):
        for r, sc in enumerate(N.schedules(p, n, inverse)):
            assert sc["signal"] == n and sc["order"] == "natural"
            passes = [s for s in sc["steps"] if s["type"] == 0]
            labels = [s["label"] for s in passes]
            core = ["x pass", "y pass", "z pass"]
            if P == 1:
                want = core if not inverse else core[::-1]
            else:
                want = ["transpose"] + core + ["landing copy"] if not inverse else ["scatter copy"] + core[::-1] + ["transpose"]
            assert labels == want, labels
            z = [s for s in passes if s["label"] == "z pass"][0]
            x0 = sc["layouts"][0][1][0]
            assert z["twiddle"] == "z" and z["tw"] == [x0, 16, 1] and z["transposed"] == 16 * 16 and z["kind"] == 1
            assert (z["A0"], z["A1"], z["B"]) == (16, 1, sc["layouts"][0][0][0])
            assert all("transposed" not in s for s in passes if s is not z)
            # peer stores: the entry rendezvous, one per exchange (three) and one between the y and z passes; all-to-all:
            # three exchanges
            rdv = sum(s["type"] == 1 for s in sc["steps"])
            a2a = sum(s["type"] == 2 for s in sc["steps"])
            assert (rdv, a2a) == ((0, 0) if P == 1 else (5, 0) if comm == 0 else (0, 3)), (rdv, a2a)


def _golden_cases():
    return [(P, comm, inverse, r) for P, comm in ((1, 0), (2, 0), (3, 0), (3, 1), (5, 0)) for inverse in (0, 1) for r in range(P)]


def test_scrambled_describe_unchanged():
    """dfft_plan_create_1d plans describe byte for byte as they did before natural order existed (the golden file holds the
    descriptions that library gave)"""
    with open(GOLDEN) as f:
        golden = json.load(f)
    n, shape = 1 << 12, (16, 16, 16)
    for P, comm, inverse, r in _golden_cases():
        p = F.plan_of(P, n, shape, comm=comm)
        with F.dry_plans(p, n, [r]) as (plan,):
            text = R.describe_raw(plan, inverse, 3)
        assert text == golden[f"P{P} comm{comm} inverse{inverse} rank{r}"], (P, comm, inverse, r)
        assert '"order"' not in text and '"transposed"' not in text


# ---- replays ------------------------------------------------------------------------------------------------------------
CASES = [
    (1, (8, 4, 16)), (2, (8, 4, 16)), (3, (8, 8, 8)), (4, (16, 8, 4)), (5, (8, 8, 16)), (6, (8, 16, 8)), (7, (8, 8, 8)),
    (8, (16, 8, 8)), (2, (2, 2, 2)), (3, (4, 4, 4)), (5, (8, 8, 8)), (6, (16, 8, 8)), (7, (16, 16, 8)),
]


def check_forward(p, n, x, got):
    """each rank's chunk is its contiguous slice of numpy.fft.fft of the flattened signal"""
    X = np.fft.fft(x.ravel())
    flat = got.ravel()
    with N.dry_plans(p, n) as plans:
        for plan in plans:
            size, start = _triple(lib().dfft_get_out_size, plan), _triple(lib().dfft_get_out_start, plan)
            lo, hi = start[0] * size[1] * size[2], (start[0] + size[0]) * size[1] * size[2]
            assert R.O.rel_l2(flat[lo:hi], X[lo:hi]) < 1e-13


@pytest.mark.parametrize("P, shape", CASES)
@pytest.mark.parametrize("comm", [0, 1])
@pytest.mark.parametrize("inverse", [0, 1])
def test_replay(P, shape, comm, inverse):
    n = int(np.prod(shape))
    assert min(shape) >= P
    p = N.plan_of(P, n, shape, comm=comm)
    if not inverse:
        x = rng_signal(shape, P)
        got = N.replay(p, n, 0, x)
        check_forward(p, n, x, got)
    else:
        x = rng_signal(shape[::-1], P)
        got = N.replay(p, n, 1, x)
    assert R.O.rel_l2(got, N.reference(x, inverse)) < 1e-13


@pytest.mark.parametrize("P", [1, 3, 5])
def test_round_trip_and_scale(P):
    shape = (8, 8, 16)
    n = int(np.prod(shape))
    x = rng_signal(shape, 7)
    p = N.plan_of(P, n, shape)
    y = N.replay(p, n, 0, x)
    back = N.replay(p, n, 1, y)
    assert R.O.rel_l2(back, n * x) < 1e-13
    ps = N.plan_of(P, n, shape, scale=(0.5, 1.0 / n))
    ys = N.replay(ps, n, 0, x)
    assert np.array_equal(ys, y * 0.5)
    assert R.O.rel_l2(N.replay(ps, n, 1, ys), 0.5 * x) < 1e-13


@pytest.mark.parametrize("P", [1, 3, 7])
def test_default_factors_replay(P):
    n = 1 << 9
    p = N.plan_of(P, n)
    assert p.shape == expected_factors(n, P)
    x = rng_signal(p.shape, 3)
    assert R.O.rel_l2(N.replay(p, n, 0, x), N.reference(x, 0)) < 1e-13
    y = rng_signal(p.shape[::-1], 4)
    assert R.O.rel_l2(N.replay(p, n, 1, y), N.reference(y, 1)) < 1e-13


def test_agrees_with_scrambled_plan():
    """the natural output is the scrambled plan's output under the scrambled index map"""
    shape, P = (8, 8, 8), 3
    n = int(np.prod(shape))
    x = rng_signal(shape, 9)
    nat = N.replay(N.plan_of(P, n, shape), n, 0, x)
    scr = F.replay(F.plan_of(P, n, shape), n, 0, x)[0]
    assert R.O.rel_l2(nat.ravel(), F.natural(scr)) < 1e-14


# ---- planted defects: the replay must catch them --------------------------------------------------------------------------
def _wrong_column(scheds):
    """every rank's z pass scatters at the next rank's column x0 instead of its own (equal slabs: no overlap, no gap)"""
    P = len(scheds)
    x0 = [sc["layouts"][0][1][0] for sc in scheds]
    for r, sc in enumerate(scheds):
        for st in sc["steps"]:
            if st.get("label") == "z pass":
                for seg in st["out"]["segs"]:
                    seg["base"] += (x0[(r + 1) % P] - x0[r]) * sc["esize"]


def _no_landing_rendezvous(scheds):
    """drop the rendezvous between the z pass and the landing copy"""
    for sc in scheds:
        k = [i for i, st in enumerate(sc["steps"]) if st.get("label") == "landing copy"][0]
        assert sc["steps"][k - 1]["type"] == 1
        del sc["steps"][k - 1]


def test_planted_wrong_column_fails():
    shape, P = (8, 8, 8), 4
    n = int(np.prod(shape))
    x = rng_signal(shape, 5)
    err = R.O.rel_l2(N.replay(N.plan_of(P, n, shape), n, 0, x, mutate=_wrong_column), N.reference(x, 0))
    assert err > 1e-2, err


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("P", [1, 3])
def test_planted_twiddle_without_k1_fails(P, inverse):
    shape = (8, 8, 8)
    n = int(np.prod(shape))
    x = rng_signal(shape, 6)
    err = R.O.rel_l2(N.replay(N.plan_of(P, n, shape), n, inverse, x, line_b=False), N.reference(x, inverse))
    assert err > 1e-2, err


def test_planted_landing_copy_without_rendezvous_fails():
    """the lock-step replay still moves the right values; the engine's slot rule catches the missing rendezvous"""
    shape, P = (8, 8, 8), 3
    n = int(np.prod(shape))
    x = rng_signal(shape, 8)
    with pytest.raises(AssertionError, match="without a rendezvous"):
        N.replay(N.plan_of(P, n, shape), n, 0, x, mutate=_no_landing_rendezvous)
