"""16-bit plans (DFFT_F16 / DFFT_BF16) without a GPU: the precisions every entry point accepts or refuses, the geometry
of 16-bit plans against the F32 plan of the same shape, the output scale split over the FFT passes, and a numpy replay of
every rank's step list with each pass's stores rounded to 16 bits (step_replay.py).

A 16-bit plan runs the F32 plan's sequential schedule with 4-byte elements: the same steps over the same element counts,
half the bytes.  Each FFT pass multiplies its stores by its "factor" (f_a = |s|^(log2 n_a / L), the sign of s on the last
FFT axis) and rounds them to nearest even."""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import lib
from oracle import dft_oracle as O
from step_replay import round16

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
C2C, R2C = dfft.C2C, dfft.R2C
F16, BF16, F32 = dfft.F16, dfft.BF16, dfft.F32
P2P, A2A = 0, 1
ERR_INVALID, ERR_UNSUPPORTED = -1, -5
SLOT_SHIFT = 44
# rel-L2 bounds against the float64 reference (about 4x one rounding per pass, u sqrt(passes) / sqrt(3))
TOL = {F16: 2e-3, BF16: 1.6e-2}


def err():
    return (lib().dfft_last_error_string() or b"").decode()


def created(p, rank=0):
    """(rc, message) of creating rank's dry plan of p, the plan destroyed again"""
    rc, msg, c, plan = R.create(p, rank)
    if rc == 0:
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return rc, msg


# ---- acceptance and refusals -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("prec", [F16, BF16])
@pytest.mark.parametrize("kw", [dict(), dict(batch=2), dict(inplace=True), dict(transform=R2C), dict(transform=R2C, inplace=True)])
def test_creators_accept_16bit(prec, kw):
    assert created(R.Plan(2, SL, (8, 8, 16), prec=prec, **kw))[0] == 0


@pytest.mark.parametrize("prec", [F16, BF16])
@pytest.mark.parametrize("what, p", [
    ("DCT / DST plans", lambda prec: R.Plan(1, SL, (8, 8, 8), transform=dfft.DCT, prec=prec)),
    ("DCT / DST plans", lambda prec: R.Plan(1, SL, (8, 8, 8), transform=dfft.DST, prec=prec)),
    ("real-to-real plans", lambda prec: R.Plan(1, SL, (8, 8, 8), kinds=(dfft.DCT, dfft.DCT, dfft.DCT), prec=prec)),
    ("padded plans", lambda prec: R.Plan(1, SL, (8, 8, 8), spectral=(4, 8, 8), prec=prec)),
    ("pruned plans", lambda prec: R.Plan(1, SL, (8, 8, 8), data=(4, 8, 8), prec=prec)),
    ("interleaved plans", lambda prec: R.Plan(1, SL, (8, 8, 8), components=2, prec=prec)),
    ("interleaved plans", lambda prec: R.Plan(1, SL, (8, 8, 8), components=1, prec=prec)),
    ("box plans", lambda prec: R.Plan(1, SL, (8, 8, 8), in_boxes=(((0, 0, 0), (8, 8, 8)),), prec=prec)),
    ("plans with strides", lambda prec: R.Plan(1, SL, (8, 8, 8), embed="in", prec=prec)),
])
def test_refused_options(prec, what, p):
    rc, msg, c, plan = R.create(p(prec), 0)
    if plan:  # strides are refused by their setter, after the plan was made
        lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    assert rc == ERR_UNSUPPORTED, (rc, msg)
    assert what in msg and "16-bit" in msg, msg


@pytest.mark.parametrize("prec", [F16, BF16])
@pytest.mark.parametrize("shape", [(6, 8, 8), (8, 12, 8), (8, 8, 5)])
def test_refused_bluestein_lengths(prec, shape):
    rc, msg = created(R.Plan(1, SL, shape, prec=prec))
    assert rc == ERR_UNSUPPORTED and "16-bit" in msg and "power-of-two" in msg, (rc, msg)
    assert created(R.Plan(1, SL, shape, prec=F32))[0] == 0  # the same shape in f32: a Bluestein plan


@pytest.mark.parametrize("prec", [4, -1, 7])
def test_bad_precision_is_invalid(prec):
    rc, msg = created(R.Plan(1, SL, (8, 8, 8), prec=prec))
    assert rc == ERR_INVALID and "bad precision" in msg
    assert lib().dfft_fft1d_contig(prec, 0, -1, 8, 1, None, 8, None, 8, None) == ERR_INVALID
    assert lib().dfft_fft1d_strided(prec, -1, 1, 8, 1, None, None, None) == ERR_INVALID


@pytest.mark.parametrize("prec", [F16, BF16])
def test_single_axis_refusals(prec):
    assert lib().dfft_fft1d_r2r(prec, dfft.DCT, -1, 8, 1, 1, None, None, None) == ERR_UNSUPPORTED
    assert "real-to-real" in err() and "16-bit" in err()
    assert lib().dfft_fft1d_contig(prec, 0, -1, 12, 1, None, 12, None, 12, None) == ERR_UNSUPPORTED
    assert lib().dfft_fft1d_strided(prec, -1, 1, 12, 1, None, None, None) == ERR_UNSUPPORTED
    s = (C.c_longlong * 3)(0, 1, 1)
    assert lib().dfft_fft1d_general(prec, -1, 5, 1, 1, 1, None, s, None, s, None) == ERR_UNSUPPORTED


def test_python_precision_names():
    for name, code in (("half", F16), ("f16", F16), ("float16", F16), ("bfloat16", BF16), ("bf16", BF16)):
        assert dfft.MPIcuFFT_Slab(dfft.Configurations(), object(), precision=name, transform="c2c").precision == code
    with pytest.raises(ValueError):
        dfft.MPIcuFFT_Slab(dfft.Configurations(), object(), precision="fp8")


# ---- geometry and step lists against the F32 plan --------------------------------------------------------------------------
CASES = [
    # P, decomp, transform, shape, p1, p2, comm, batch, inplace, axes
    (1, SL, C2C, (8, 16, 32), 1, 1, P2P, None, False, None),
    (1, SL, R2C, (4, 8, 64), 1, 1, P2P, None, True, None),
    (2, SL, R2C, (8, 8, 32), 2, 1, A2A, None, False, None),
    (3, SL, C2C, (8, 16, 16), 3, 1, P2P, None, False, None),          # uneven split
    (4, SL, C2C, (16, 8, 64), 4, 1, P2P, 2, False, None),             # peer stores, batch 2
    (4, SL, R2C, (8, 16, 128), 4, 1, P2P, None, False, None),         # blocked hand-over + tail column
    (4, ZY, C2C, (8, 4, 16), 4, 1, A2A, None, True, None),
    (4, ZY, R2C, (8, 4, 32), 4, 1, P2P, None, True, None),
    (6, PE, C2C, (8, 16, 32), 2, 3, P2P, None, False, None),          # uneven pencil split
    (8, PE, R2C, (8, 16, 32), 2, 4, A2A, None, True, None),
    (8, PE, C2C, (16, 8, 32), 4, 2, P2P, 2, False, None),
    (4, PE, C2C, (8, 16, 32), 2, 2, P2P, None, False, (0, 1, 1)),     # kept x axis
    (2, SL, R2C, (8, 16, 32), 2, 1, P2P, None, False, (1, 0, 1)),     # kept y axis
]
IDS = [f"P{c[0]}-{'sl zy pe'.split()[c[1]]}-{'r2c' if c[2] == R2C else 'c2c'}-{'x'.join(map(str, c[3]))}" + ("-b2" if c[7] else "") +
       ("-ip" if c[8] else "") + (f"-axes{''.join(map(str, c[9]))}" if c[9] else "") for c in CASES]


def plan_of(case, prec, scale=None):
    P, decomp, transform, shape, p1, p2, comm, batch, inplace, axes = case
    return R.Plan(P, decomp, shape, p1, p2, transform=transform, prec=prec, comm=comm, batch=batch, inplace=inplace, axes=axes, scale=scale)


def normalized(sc):
    """the step list with addresses in elements: slot views as (rank, slot, element), caller views as element offsets"""
    es, sb = sc["esize"], sc["slot_bytes"]

    def base(b):
        if b >> SLOT_SHIFT:
            off = b & ((1 << SLOT_SHIFT) - 1)
            assert (off % sb) % es == 0
            return ((b >> SLOT_SHIFT) - 1, off // sb, (off % sb) // es)
        assert b % es == 0
        return b // es

    steps = []
    for st in sc["steps"]:
        st = dict(st)
        st.pop("factor", None)
        for w in ("in", "out"):
            if w in st:
                st[w] = {**st[w], "segs": [{**g, "base": base(g["base"])} for g in st[w]["segs"]]}
        steps.append(st)
    return steps


@pytest.mark.parametrize("d", [1, 2, 3])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_geometry_matches_f32(case, d):
    P = case[0]
    for prec in (F16, BF16):
        for inverse in (0, 1):
            with R.dry_plans(plan_of(case, prec)) as half, R.dry_plans(plan_of(case, F32)) as full:
                for r in range(P):
                    a, b = R.schedule(plan_of(case, prec), half[r], inverse, d), R.schedule(plan_of(case, F32), full[r], inverse, d)
                    assert a["esize"] == 4 and b["esize"] == 8
                    assert a["precision"] == ("f16" if prec == F16 else "bf16") and "precision" not in b
                    assert not a["overlapped"] and not b["overlapped"]
                    assert 2 * a["domain_bytes"] == b["domain_bytes"]
                    assert a["nslots"] == b["nslots"]
                    assert a["slot_bytes"] % 256 == 0 and b["slot_bytes"] // 2 <= a["slot_bytes"] < b["slot_bytes"] // 2 + 256
                    assert a["work_bytes"] == a["nslots"] * a["slot_bytes"]
                    assert a["layouts"] == b["layouts"]
                    if "field_in" in b:
                        assert (2 * a["field_in"], 2 * a["field_out"]) == (b["field_in"], b["field_out"])
                    assert normalized(a) == normalized(b)
                    assert not any("factor" in st or "scale" in st for st in a["steps"])  # s = 1: unscaled


def fft_passes(sc):
    return [st for st in sc["steps"] if st["type"] == 0 and st["kind"] not in (6, 7)]


def axis_length(st):
    return 1 << (st["log2n"] + (1 if st["kind"] in (2, 3) else 0))  # R2C / C2R: Nz reals, log2n of Nz / 2 pairs


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_factors_of_forward_normalisation(case):
    """s = 1/N: every FFT pass stores times exactly 1/n_a, copies never scale, no pass carries "scale"."""
    for d in (1, 2, 3):
        for inverse in (0, 1):
            # the axes the exec transforms: those of its FFT passes (each label names its axis)
            with R.dry_plans(plan_of(case, F16)) as (plan, *_):
                labels = {st["label"][0] for st in fft_passes(R.schedule(plan_of(case, F16), plan, inverse, d))}
            assert labels <= set("xyz")
            s = 1.0 / math.prod(case[3]["xyz".index(a)] for a in labels)
            p = plan_of(case, F16, (1.0, s) if inverse else (s, 1.0))
            with R.dry_plans(p) as plans:
                for plan in plans:
                    sc = R.schedule(p, plan, inverse, d)
                    for st in sc["steps"]:
                        assert "scale" not in st
                        if st["type"] == 0 and st["kind"] in (6, 7):
                            assert "factor" not in st
                    for st in fft_passes(sc):
                        assert st["factor"] == 1.0 / axis_length(st), (st["label"], st.get("factor"))


@pytest.mark.parametrize("case", [c for c in CASES if c[3][0] != c[3][1] != c[3][2] != c[3][0] and c[9] is None], ids=lambda c: f"P{c[0]}-{c[3]}")
def test_sign_on_last_axis_only(case):
    """s = -3: the factors multiply to |s| per output value, and the steps of the exec's last FFT axis alone are negative"""
    for inverse in (0, 1):
        p = plan_of(case, BF16, (1.0, -3.0) if inverse else (-3.0, 1.0))
        with R.dry_plans(p) as plans:
            for plan in plans:
                passes = fft_passes(R.schedule(p, plan, inverse, 3))
                last = axis_length(passes[-1])
                per_axis = {}
                for st in passes:
                    assert (st["factor"] < 0) == (axis_length(st) == last), st["label"]
                    per_axis[axis_length(st)] = abs(st["factor"])
                assert len(per_axis) == 3
                assert math.prod(per_axis.values()) == pytest.approx(3.0, rel=1e-6)
                L = sum(int(math.log2(n)) for n in per_axis)
                for n, f in per_axis.items():
                    assert f == float(np.float32(3.0 ** (math.log2(n) / L)))


def test_no_axis_transformed_moves_unscaled():
    p = R.Plan(2, SL, (8, 8, 16), prec=F16, axes=(0, 0, 0), scale=(0.5, 0.25))
    for inverse in (0, 1):
        with R.dry_plans(p) as plans:
            for plan in plans:
                sc = R.schedule(p, plan, inverse, 3)
                assert not fft_passes(sc) and not any("factor" in st or "scale" in st for st in sc["steps"])


# ---- numpy replay with 16-bit rounding ------------------------------------------------------------------------------------
def replay_case(case, prec, inverse, d, scale):
    P, decomp, transform, shape, *_ = case
    axes = case[9] or (1, 1, 1)
    p = plan_of(case, prec, scale)
    c2c = transform == C2C
    fields = p.fields
    # the oracle's values lie in [0, 256): shifted and scaled to [-1, 1), so that unnormalised small transforms fit FP16
    xs = [(O.complex_input(shape, seed=7 + f) - (128 + 128j)) / 128 if c2c else O.real_input(shape, seed=7 + f) / 128 - 1 for f in range(fields)]
    tr = [a for a in (2, 1, 0)[:d] if axes[a]]

    def fwd(x):
        X = np.asarray(x, dtype=np.complex128)
        if not c2c:
            X = np.fft.rfft(x, axis=2)
            return np.fft.fftn(X, axes=[a for a in tr if a != 2]) if len(tr) > 1 else X
        return np.fft.fftn(X, axes=tr) if tr else X

    def inv(X):
        if c2c:
            return np.fft.ifftn(X, axes=tr) * math.prod(shape[a] for a in tr) if tr else X
        Y = np.fft.ifftn(X, axes=[a for a in tr if a != 2]) * math.prod(shape[a] for a in tr if a != 2) if len(tr) > 1 else X
        return np.fft.irfft(Y, n=shape[2], axis=2) * shape[2]

    if inverse:
        ins = [round16(fwd(x) / math.prod(shape[a] for a in tr), prec) for x in xs]
        want = [scale[1] * inv(X) for X in ins]
    else:
        ins = [round16(x, prec) for x in xs]
        want = [scale[0] * fwd(x) for x in ins]
    outs = R.replay(p, inverse, d, ins)
    return R.error(outs, want)


@pytest.mark.parametrize("prec", [F16, BF16], ids=["f16", "bf16"])
@pytest.mark.parametrize("case", [c for c in CASES if c[9] is None or c[2] == C2C], ids=lambda c: f"P{c[0]}-{'sl zy pe'.split()[c[1]]}-{'r2c' if c[2] == R2C else 'c2c'}-{'x'.join(map(str, c[3]))}")
def test_replay_with_16bit_rounding(case, prec):
    n = math.prod(case[3])
    for inverse, d, scale in ((0, 3, (1.0, 1.0)), (0, 3, (1.0 / n, 1.0)), (1, 3, (1.0, 1.0)), (1, 3, (1.0, 0.5)), (0, 1, (1.0, 1.0)),
                              (1, 2, (1.0, 1.0))):
        if (case[9] is not None and d < 3) or (case[1] == ZY and inverse and d == 2):  # ZY's inverse d = 2 runs its x pass as well
            continue
        e = replay_case(case, prec, inverse, d, scale)
        assert e < TOL[prec], (inverse, d, scale, e)


def test_rounding_helper_is_round_to_nearest_even():
    # bfloat16: 1 + 2^-8 is a tie between 1 and 1 + 2^-7, and rounds to the even 1; 1 + 3 * 2^-8 to 1 + 2^-6
    assert round16(np.array([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8]), BF16).tolist() == [1.0, 1 + 2.0 ** -6]
    assert round16(np.array([1 + 2.0 ** -11]), F16).tolist() == [1.0]
