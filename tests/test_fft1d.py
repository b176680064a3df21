"""Distributed 1D complex transforms (dfft_plan_create_1d) without a GPU: refusals, the default factors, describe keys, the
two-level twiddle table, and replays of every rank's step list on geometry-only communicators against numpy.fft.fft of the
flattened signal under the scrambled index map."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np
import pytest

import fft1d_replay as F
import step_replay as R
import distributedfft_b200 as dfft
from distributedfft_b200._lib import check, lib

SLAB = dfft.SLAB_ZY_THEN_X
ERR_INVALID, ERR_UNSUPPORTED = -1, -5


def rng_signal(shape, seed=0):
    g = np.random.default_rng(seed)
    return g.standard_normal(shape) + 1j * g.standard_normal(shape)


def create_rc(P, n, factors=None, prec=dfft.F64, rank=0):
    rc, msg, c, plan = F.create(R.Plan(P, SLAB, (0, 0, 0), prec=prec), n, factors, rank)
    if rc == 0:
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return rc, msg


@pytest.mark.parametrize("P, n, factors, prec, code, text", [
    (1, 1 << 10, None, dfft.F16, ERR_UNSUPPORTED, "1D plans have no 16-bit storage"),
    (1, 1 << 10, None, dfft.BF16, ERR_UNSUPPORTED, "1D plans have no 16-bit storage"),
    (1, 1000, None, dfft.F64, ERR_UNSUPPORTED, "power of two in [8, 2^39]"),
    (1, 4, None, dfft.F64, ERR_UNSUPPORTED, "power of two in [8, 2^39]"),
    (1, 1 << 40, None, dfft.F64, ERR_UNSUPPORTED, "power of two in [8, 2^39]"),
    (1, 1 << 15, (1 << 14, 1, 2), dfft.F64, ERR_UNSUPPORTED, "powers of two in [2, 8192]"),
    (1, 1 << 15, (6, 64, 64), dfft.F64, ERR_UNSUPPORTED, "powers of two in [2, 8192]"),
    (1, 1 << 15, (32, 32, 16), dfft.F64, ERR_INVALID, "multiply to n"),
    (4, 1 << 12, (2, 64, 32), dfft.F64, ERR_INVALID, "at least the rank count"),
    (4, 1 << 12, (64, 2, 32), dfft.F64, ERR_INVALID, "at least the rank count"),
    (16, 1 << 5, None, dfft.F64, ERR_UNSUPPORTED, "has no split into three powers of two"),
    (1, 1 << 10, None, 9, ERR_INVALID, "bad precision"),
])
def test_create_refusals(P, n, factors, prec, code, text):
    rc, msg = create_rc(P, n, factors, prec)
    assert rc == code and text in msg, (rc, msg)


def test_default_factor_split_refused():
    # 16 ranks need N1, N2 >= 16: 2^8 * 2^1 = 512 points at least
    rc, msg = create_rc(16, 1 << 8)
    assert rc == ERR_UNSUPPORTED and "has no split" in msg, (rc, msg)
    assert create_rc(16, 1 << 9)[0] == 0


def expected_factors(n, P):
    """the factor rule of dfft.h, or None where no split exists"""
    L, lp = n.bit_length() - 1, max(1, (P - 1).bit_length())
    cands = [(l1, l2, L - l1 - l2) for l1 in range(lp, 14) for l2 in range(lp, 14) if 1 <= L - l1 - l2 <= 13]
    if not cands:
        return None
    l1, l2, l3 = min(cands, key=lambda c: (max(c) - min(c), -c[0], -c[1]))
    return 1 << l1, 1 << l2, 1 << l3


@pytest.mark.parametrize("P", [1, 2, 3, 5, 8])
def test_default_factors(P):
    for L in range(3, 40):
        n = 1 << L
        rc, msg, c, plan = F.create(R.Plan(P, SLAB, (0, 0, 0)), n, None, 0)
        if rc:
            assert rc == ERR_UNSUPPORTED and expected_factors(n, P) is None, (L, P, msg)
            lib().dfft_comm_destroy(c)
            continue
        f = F.factors_of(plan)
        assert f == expected_factors(n, P) and f[0] * f[1] * f[2] == n and min(f[:2]) >= P, (L, P, f)
        if P == 1:  # as balanced as powers of two allow
            assert max(f).bit_length() - min(f).bit_length() <= 1, (L, f)
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)


def test_setter_and_exec_refusals():
    rc, msg, c, plan = F.create(R.Plan(1, SLAB, (0, 0, 0)), 1 << 12, None, 0)
    assert rc == 0, msg
    try:
        assert lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(0, 1, 1)) == ERR_UNSUPPORTED
        assert "1D plans transform every axis" in lib().dfft_last_error_string().decode()
        assert lib().dfft_plan_set_strides(plan, (C.c_longlong * 3)(4096, 256, 16), None) == ERR_UNSUPPORTED
        assert "1D plans" in lib().dfft_last_error_string().decode()
        assert lib().dfft_plan_set_weights(plan, (C.c_void_p * 3)(None, None, 1 << 40)) == ERR_UNSUPPORTED
        assert "1D plans have no spectral weights" in lib().dfft_last_error_string().decode()
        for d in (1, 2):
            need = C.c_size_t()
            assert lib().dfft_plan_describe(plan, 0, d, None, 0, C.byref(need)) == ERR_UNSUPPORTED
            assert "d = 3" in lib().dfft_last_error_string().decode()
        f = (C.c_size_t * 3)()
        assert lib().dfft_plan_get_1d_factors(None, f) == ERR_INVALID
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)
    p = R.Plan(1, SLAB, (16, 16, 16))
    with R.dry_plans(p) as (plan3d,):
        assert lib().dfft_plan_get_1d_factors(plan3d, (C.c_size_t * 3)()) == ERR_INVALID
        assert "signal" not in json.loads(R.describe_raw(plan3d, 0, 3))


def test_python_binding_refusals():
    """the binding refuses what 1D plans do not take before it creates a plan (no device needed)"""
    def binding(cls, transform):
        p = cls.__new__(cls)
        p.config, p.precision, p.kinds, p.transform = dfft.Configurations(), dfft.F64, None, transform
        p.comm = type("DryComm", (), {"size": 1, "_h": None})()
        return p

    slab = binding(dfft.MPIcuFFT_Slab, dfft.C2C)
    for args, kw in (((None,), {"batch": 2}), ((dfft.GlobalSize(16, 16, 16),), {}), ((None,), {"transform_axes": (False, True, True)}),
                     ((None, dfft.Partition(1, 1)), {}), ((None,), {"in_strides": (4096, 256, 16)}), ((None, None, False), {})):
        with pytest.raises(ValueError, match="1D plans are C2C"):
            slab.initFFT(*args, signal=1 << 12, **kw)
    for kw in ({"inplace": True}, {"spectral": (4, 4, 4)}, {"components": 2}, {"data": (4, 4, 4)}):
        with pytest.raises(ValueError, match="1D plans are out of place"):
            slab.initFFT(None, signal=1 << 12, **kw)
    with pytest.raises(ValueError, match="factors belong to a 1D plan"):
        slab.initFFT(dfft.GlobalSize(16, 16, 16), factors=(16, 16, 16))
    with pytest.raises(ValueError, match="1D plans are C2C"):
        binding(dfft.MPIcuFFT_Slab, dfft.R2C).initFFT(None, signal=1 << 12)
    with pytest.raises(ValueError, match="slab plans"):
        binding(dfft.MPIcuFFT_Slab_Z_Then_YX, dfft.C2C).initFFT(None, signal=1 << 12)


@pytest.mark.parametrize("P, comm", [(1, 0), (3, 0), (3, 1)])
def test_describe_keys(P, comm):
    p = F.plan_of(P, 1 << 12, (16, 16, 16), comm=comm)
    for inverse in (0, 1):
        for r in range(P):
            sc = F.schedules(p, 1 << 12, inverse)[r]
            assert sc["signal"] == 1 << 12
            passes = [s for s in sc["steps"] if s["type"] == 0]
            labels = [s["label"] for s in passes]
            core = ["x pass", "y pass", "z pass"]
            want = (["transpose"] if P > 1 else []) + core if not inverse else core[::-1] + (["transpose"] if P > 1 else [])
            assert labels == want, labels
            tw = {s["label"]: (s.get("twiddle"), s.get("tw")) for s in passes}
            x0 = sc["layouts"][0][1][0]
            assert tw["y pass"] == ("y", [x0, 0, 16]) and tw["z pass"] == ("z", [x0, 16, 1])
            assert tw["x pass"] == (None, None) and all(s["inverse"] == inverse for s in passes)
            # every layout of a 1D plan is the rank's x-slab
            assert all(l == sc["layouts"][0] for l in sc["layouts"])


# ---- the two-level twiddle table ----------------------------------------------------------------------------------------
def two_level(L, m, dtype):
    """W_N^m, N = 2^L, as the kernels form it from the table entries rounded to dtype (dfft_plan.cu make_tw1d_table)"""
    lo = (L + 1) // 2
    m = np.asarray(m, dtype=np.uint64) & np.uint64((1 << L) - 1)
    ml, mh = m & np.uint64((1 << lo) - 1), m >> np.uint64(lo)
    two_pi = np.longdouble(2) * np.longdouble(np.pi)  # np.pi in long double is not exact: use the angle's own rounding
    two_pi = np.longdouble("6.28318530717958647692528676655900577")
    a_lo = -two_pi * ml.astype(np.longdouble) / np.longdouble(2) ** L
    a_hi = -two_pi * mh.astype(np.longdouble) / np.longdouble(2) ** (L - lo)
    t_lo = (np.cos(a_lo) + 1j * np.sin(a_lo)).astype(dtype)
    t_hi = (np.cos(a_hi) + 1j * np.sin(a_hi)).astype(dtype)
    return t_hi * t_lo  # the product in the working precision, as cmul does


@pytest.mark.skipif(np.finfo(np.longdouble).eps > 1e-18, reason="needs an x87 long double")
@pytest.mark.parametrize("dtype, bound", [(np.complex128, 4e-16), (np.complex64, 3e-7)])
def test_twiddle_table_long_double(dtype, bound):
    g = np.random.default_rng(1)
    two_pi = np.longdouble("6.28318530717958647692528676655900577")
    for L in (3, 10, 20, 27, 30, 33, 39):
        N = 1 << L
        m = np.concatenate([np.arange(min(N, 64)), N - 1 - np.arange(min(N, 64)), g.integers(0, N, 4096, dtype=np.uint64)]).astype(np.uint64)
        got = two_level(L, m, dtype).astype(np.clongdouble)
        a = -two_pi * m.astype(np.longdouble) / np.longdouble(N)
        exact = np.cos(a) + 1j * np.sin(a)
        err = np.abs(got - exact).max()
        assert err < bound, (L, float(err))


# ---- replays ------------------------------------------------------------------------------------------------------------
CASES = [
    (1, (8, 4, 16)), (2, (8, 4, 16)), (3, (8, 8, 8)), (4, (16, 8, 4)), (5, (8, 8, 16)), (6, (8, 16, 4)), (7, (8, 8, 8)),
    (8, (16, 8, 8)), (2, (2, 2, 2)), (3, (4, 4, 2)),
]


@pytest.mark.parametrize("P, shape", CASES)
@pytest.mark.parametrize("comm", [0, 1])
@pytest.mark.parametrize("inverse", [0, 1])
def test_replay(P, shape, comm, inverse):
    if shape[0] < P or shape[1] < P:
        pytest.skip("N1 and N2 below the rank count")
    n = int(np.prod(shape))
    p = F.plan_of(P, n, shape, comm=comm)
    x = rng_signal(shape, P)
    got = F.replay(p, n, inverse, x)[0]
    err = R.O.rel_l2(got, F.reference(x, inverse))
    assert err < 1e-13, err


@pytest.mark.parametrize("P", [1, 3, 5])
def test_round_trip_and_scale(P):
    shape = (8, 8, 16)
    n = int(np.prod(shape))
    x = rng_signal(shape, 7)
    p = F.plan_of(P, n, shape)
    y = F.replay(p, n, 0, x)[0]
    back = F.replay(p, n, 1, y)[0]
    assert R.O.rel_l2(back, n * x) < 1e-13
    ps = F.plan_of(P, n, shape, scale=(0.5, 1.0 / n))
    ys = F.replay(ps, n, 0, x)[0]
    assert np.array_equal(ys, y * 0.5)
    assert R.O.rel_l2(F.replay(ps, n, 1, ys)[0], 0.5 * x) < 1e-13


@pytest.mark.parametrize("P", [1, 3])
def test_default_factors_replay(P):
    n = 1 << 9
    p = F.plan_of(P, n)
    assert p.shape == expected_factors(n, P)
    x = rng_signal(p.shape, 3)
    for inverse in (0, 1):
        assert R.O.rel_l2(F.replay(p, n, inverse, x)[0], F.reference(x, inverse)) < 1e-13


# ---- planted defects: the replay must catch them --------------------------------------------------------------------------
def _shift_line0(delta=0, zero=False, label="y pass"):
    def mutate(scheds):
        for sc in scheds:
            for st in sc["steps"]:
                if st.get("label") == label and "tw" in st:
                    st["tw"][0] = 0 if zero else st["tw"][0] + delta
    return mutate


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("defect", ["k1 off by one", "no rank offset", "z k1 off by one"])
def test_planted_defects_fail(inverse, defect):
    shape, P = (8, 8, 8), 3
    n = int(np.prod(shape))
    p = F.plan_of(P, n, shape)
    x = rng_signal(shape, 5)
    mutate = {"k1 off by one": _shift_line0(1), "no rank offset": _shift_line0(zero=True),
              "z k1 off by one": _shift_line0(1, label="z pass")}[defect]
    err = R.O.rel_l2(F.replay(p, n, inverse, x, mutate=mutate)[0], F.reference(x, inverse))
    assert err > 1e-2, (defect, err)


def test_planted_unconjugated_inverse_fails():
    shape, P = (8, 8, 8), 2
    n = int(np.prod(shape))
    p = F.plan_of(P, n, shape)
    x = rng_signal(shape, 6)
    err = R.O.rel_l2(F.replay(p, n, 1, x, conj=False)[0], F.reference(x, 1))
    assert err > 1e-2, err
