"""Replays multi-rank schedules on one GPU with the real pass kernels.

The CPU replays (test_schedule_emulation and the family replays) check the data movement of every rank's step list with
numpy in place of the kernels.  Here the same step lists run on one H100 through dfft_debug_run_step (gpu_replay.py): every
rank gets its own work area and user buffers, the ranks run in lock step (pass steps through the hook, all-to-all steps as
device copies, rendezvous as no-ops), so the multi-rank kernel paths execute — multi-segment views, stores into other ranks' slots with the
blocked hand-over and its tail columns, grid-limited launches of the overlapped schedules, R2R line pairing on rank-local
counts.  Every case is checked three ways:
  1. bit for bit against the one-rank plan of the same transform on the whole grid (R2R plans excepted, see below);
  2. against a long-double reference: rel-L2 <= 3 u sqrt(sum log2 L) and max |err| <= 10 times that times rms(ref), u the
     unit roundoff of the plan's precision and L the power-of-two length each transformed axis runs (M for Bluestein axes);
  3. the inputs are unchanged and no output element is still the NaN every buffer starts as.
Each case runs twice, the ranks of a step in ascending and in descending order, and both runs must agree bit for bit: a
same-step hazard between ranks shows up as a difference.

Worst errors measured over this module on an H100 80GB HBM3 (700 W), in units of u sqrt(sum log2 L), rel-L2 / max over
rms(ref): C2C 0.66 / 3.4 (f64), 0.68 / 3.2 (f32); R2C / C2R 0.67 / 4.0, 0.67 / 4.7; Bluestein 1.03 / 4.8, 1.11 / 4.4;
R2R 0.69 / 3.7, 0.70 / 3.3; plans with kept axes 0.58 / 2.8, 0.53 / 2.0.  The bounds (3 and 30) hold every family."""
import ctypes as C
import math
import random
from dataclasses import replace

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
import step_replay as R
from distributedfft_b200._lib import check, lib
from gpu_replay import assemble, caller_buffers, element_type, nan_buffer, output, replay, run_step, same_bits, work_offset
from step_replay import view_indices
from test_inplace import run_inplace
from test_schedule_emulation import CASES, KNOBS, random_case, run_case
from test_transform_axes import fwd_ref, inv_ref, run as replay_cpu

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
C2C, R2C, DCT, DST, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.DST, dfft.R2HC
F32, F64 = dfft.F32, dfft.F64
ERR_INVALID, ERR_UNSUPPORTED = -1, -5
UNIT = {F64: 2.0 ** -53, F32: 2.0 ** -24}
WORST = {}  # (family, precision) -> worst measured (rel-L2, max) error in units of u sqrt(sum log2 L)


def case(P, decomp, transform, shape, p1, p2, comm=P2P, send=SYNC, inverse=0, d=3, prec=F64, kinds=None, axes=None, batch=None,
         inplace=False, scale=None, env=None):
    """(plan, inverse, d, environment) of one replay"""
    p = R.Plan(P, decomp, tuple(shape), p1, p2, transform=transform, kinds=kinds, prec=prec, comm=comm, send=send, batch=batch,
               inplace=inplace, axes=axes, scale=scale)
    return p, inverse, d, env or {}


def kinds_of(p):
    """the per-axis R2R kinds of p, None for C2C and R2C plans"""
    return p.kinds if p.kinds is not None or p.transform in (C2C, R2C) else (p.transform,) * 3


def geometry(p, d):
    """the fields error_check and run_lengths read"""
    return dict(prec=p.prec, shape=p.shape, d=d, axes=p.axes or (1, 1, 1))


# ---- inputs and the long-double reference ----------------------------------------------------------------------------------
def global_input(p, inverse, d, seed):
    """(input in the plan's precision, the same values in long double) of shape (batch, ...) — zero-mean normal; an inverse
    R2C input is the forward transform of real normal data, so that it is the spectrum of a real array"""
    rng = np.random.default_rng(seed)
    nx, ny, nz = p.shape
    b = p.fields
    real = kinds_of(p) is not None
    cplx_dt, real_dt = (np.complex128, np.float64) if p.prec == F64 else (np.complex64, np.float32)
    if inverse and p.transform == R2C and not real:
        x = rng.standard_normal((b, nx, ny, nz)).astype(np.longdouble)
        X = np.stack([fwd_ref(x[f], R2C, None, p.axes or (1, 1, 1), d) for f in range(b)]).astype(cplx_dt)
        return X, X.astype(np.clongdouble)
    shape = (b, nx, ny, nz)
    if real or (p.transform == R2C and not inverse):
        x = rng.standard_normal(shape).astype(real_dt)
        return x, x.astype(np.longdouble)
    x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cplx_dt)
    return x, x.astype(np.clongdouble)


def reference(p, inverse, d, x_ld):
    kinds = kinds_of(p)
    t = p.transform if kinds is None else None
    axes = p.axes or (1, 1, 1)
    if inverse:
        y = np.stack([inv_ref(x_ld[f], t, kinds, axes, d, p.shape[2]) for f in range(p.fields)])
    else:
        y = np.stack([fwd_ref(x_ld[f], t, kinds, axes, d) for f in range(p.fields)])
    sc = 1.0 if p.scale is None else p.scale[1 if inverse else 0]
    if p.prec == F32:
        sc = float(np.float32(sc))
    return y * np.longdouble(sc)


def run_lengths(s):
    """the power-of-two length each transformed axis among the first d runs (M for Bluestein axes)"""
    out = []
    for axis in (2, 1, 0)[:s["d"]]:
        if s["axes"][axis]:
            n = s["shape"][axis]
            out.append(n if n & (n - 1) == 0 else 1 << (2 * n - 2).bit_length())
    return out


def family(p, d):
    axes = p.axes or (1, 1, 1)
    if any(not axes[a] for a in (2, 1, 0)[:d]):
        return "copy"
    if kinds_of(p) is not None:
        return "R2R"
    if any(p.shape[a] & (p.shape[a] - 1) for a in (2, 1, 0)[:d] if axes[a]):
        return "Bluestein"
    return "R2C/C2R" if p.transform == R2C else "C2C"


def error_check(s, got, want, extra=None):
    """check 2 (s: the fields of geometry()); returns (rel-L2, max) in units of u sqrt(sum log2 L)"""
    unit = UNIT[s["prec"]] * math.sqrt(max(1.0, sum(math.log2(n) for n in run_lengths(s))))
    want = np.asarray(want)
    err = got.astype(want.dtype) - want
    if extra is not None:
        err = err + extra
    ref_norm = float(np.sqrt(np.sum(np.abs(want) ** 2)))
    rel = float(np.sqrt(np.sum(np.abs(err) ** 2))) / ref_norm
    rms = ref_norm / math.sqrt(want.size)
    mx = float(np.max(np.abs(err))) / rms
    return rel / unit, mx / unit


# ---- the replay -------------------------------------------------------------------------------------------------------------
def one_rank_plan(p, comm):
    """the real one-rank plan of p's transform on the whole grid, every setter applied"""
    rc, msg, _, plan = R.create(replace(p, P=1, p1=1, p2=1), 0, comm)
    assert rc == 0, msg
    R.set_options(p, plan)
    return plan


def one_rank(p, inverse, d, x):
    """the real one-rank plan of the same transform on the whole grid: its output (batch, ...)"""
    comm = C.c_void_p()
    check(lib().dfft_comm_create(0, 1, None, torch.cuda.current_device(), C.byref(comm)))
    plan = one_rank_plan(p, comm)
    try:
        real = kinds_of(p) is not None
        es = (8 if real else 16) // (1 if p.prec == F64 else 2)  # bytes per view element
        sc = {"esize": es, "domain_bytes": lib().dfft_get_domain_size(plan), "layouts": R.layouts(plan)}
        if real:
            sc["r2r"] = True
        _, so, bi, bo, _ = caller_buffers(p, sc, inverse, d, x)
        torch.cuda.synchronize()
        direction = 1 if inverse else -1
        if real:
            check(lib().dfft_exec_r2r_partial(plan, bo.data_ptr(), bi.data_ptr(), direction, d))
        elif p.transform == C2C:
            check(lib().dfft_exec_c2c_partial(plan, bo.data_ptr(), bi.data_ptr(), direction, d))
        elif inverse:
            check(lib().dfft_exec_c2r_partial(plan, bo.data_ptr(), bi.data_ptr(), d))
        else:
            check(lib().dfft_exec_r2c_partial(plan, bo.data_ptr(), bi.data_ptr(), d))
        got = bo.cpu().numpy().view(element_type(sc))
        return np.stack([so.get(got, f) for f in range(p.fields)])
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(comm)


def check_case(p, inverse, d, seed=0):
    x, x_ld = global_input(p, inverse, d, seed)
    # 3: no element left unwritten, the inputs intact, the same bits with the ranks of each step in the other order
    got = output(p, inverse, d, x)
    # 1: the one-rank plan on the whole grid
    if p.kinds is None:
        want1 = one_rank(p, inverse, d, x)
        assert same_bits(got, want1), f"differs from the one-rank plan at {np.argwhere(got != want1)[:8].tolist()}"
    # else: R2R passes transform lines in pairs (two real lines as one complex line), and which lines pair up follows the
    # rank-local line and column counts, so the rounding differs from the one-rank plan's; check 2 covers them
    # 2: the long-double reference
    ref = reference(p, inverse, d, x_ld)
    rel, mx = error_check(geometry(p, d), got, ref)
    key = (family(p, d), "f64" if p.prec == F64 else "f32")
    WORST[key] = (max(WORST.get(key, (0, 0))[0], rel), max(WORST.get(key, (0, 0))[1], mx))
    assert rel <= 3.0, f"rel-L2 error {rel:.2f} u sqrt(sum log2 L)"
    assert mx <= 30.0, f"max error {mx:.2f} u sqrt(sum log2 L) rms(ref)"
    return got, ref


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    if WORST:
        print("\nworst error per family, in u sqrt(sum log2 L) (rel-L2 bound 3, max bound 30):")
        for (fam, prec), (rel, mx) in sorted(WORST.items()):
            print(f"  {fam:10s} {prec}: rel-L2 {rel:.3f}  max {mx:.3f}")


@pytest.fixture
def knobs(monkeypatch):
    def apply(env):
        for k in KNOBS:
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
    return apply


# ---- cases --------------------------------------------------------------------------------------------------------------------
MIXED = (R2HC, DST, DCT)
EXTRA = [  # powers of two except for the Bluestein cases: odd rank counts make the splits uneven
    # uneven splits on 2, 3, 5, 6, 7 and 8 ranks, every decomposition and method
    case(2, SL, C2C, (8, 32, 64), 2, 1, A2A),
    case(3, SL, R2C, (16, 16, 64), 3, 1, P2P, STREAMS),
    case(5, SL, C2C, (16, 16, 128), 5, 1, P2P),
    case(5, ZY, R2C, (16, 8, 64), 5, 1, A2A),
    case(7, ZY, C2C, (16, 8, 64), 7, 1, P2P),
    case(6, PE, C2C, (16, 16, 32), 3, 2, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    case(6, PE, R2C, (8, 16, 64), 2, 3, A2A),
    case(7, PE, C2C, (16, 8, 32), 7, 1, P2P),  # P2 = 1
    case(7, PE, R2C, (8, 16, 64), 1, 7, P2P),  # P1 = 1
    case(8, PE, R2C, (16, 8, 128), 4, 2, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    case(8, SL, C2C, (32, 16, 64), 8, 1, P2P, STREAMS),
    case(3, PE, C2C, (16, 16, 32), 3, 1, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    case(5, SL, R2C, (16, 32, 128), 5, 1, P2P, STREAMS, env={"DFFT_XCHG_CTAS": "32"}),
    # partial d
    case(6, PE, R2C, (8, 16, 64), 3, 2, P2P, d=1),
    case(6, PE, C2C, (16, 8, 64), 2, 3, A2A, d=2),
    # long axes: wide tiles and the TMA-fed kernel on single-segment local passes
    case(2, SL, C2C, (8, 16, 8192), 2, 1, P2P),
    case(4, PE, R2C, (16, 8, 4096), 2, 2, P2P),
    case(3, SL, C2C, (8, 1024, 32), 3, 1, A2A),
    case(4, ZY, C2C, (2048, 8, 16), 4, 1, P2P),
    case(8, PE, C2C, (1024, 16, 32), 2, 4, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    # R2C with odd Nzc tails
    case(3, SL, R2C, (8, 16, 256), 3, 1, P2P),  # Nzc = 129
    case(5, PE, R2C, (16, 16, 32), 1, 5, P2P),  # Nzc = 17 over 5
    # Bluestein lengths
    case(3, SL, C2C, (96, 100, 90), 3, 1, P2P),
    case(4, PE, C2C, (12, 30, 27), 2, 2, A2A),
    case(5, ZY, C2C, (20, 24, 45), 5, 1, P2P),
    # DCT, DST and mixed kinds with odd rank-local counts
    case(3, SL, None, (16, 8, 32), 3, 1, P2P, kinds=(DCT, DCT, DCT)),
    case(5, PE, None, (16, 16, 16), 1, 5, A2A, kinds=(DST, DST, DST)),
    case(6, PE, None, (8, 16, 32), 3, 2, P2P, kinds=MIXED),
    case(7, ZY, None, (16, 8, 32), 7, 1, P2P, kinds=(DCT, R2HC, DST)),
    # kept axes (copy passes)
    case(4, PE, C2C, (8, 16, 32), 2, 2, P2P, axes=(0, 1, 1)),
    case(3, SL, R2C, (8, 8, 32), 3, 1, A2A, axes=(1, 0, 1)),
    case(5, ZY, None, (16, 8, 16), 5, 1, P2P, kinds=MIXED, axes=(1, 1, 0)),
    case(6, PE, C2C, (8, 16, 16), 3, 2, P2P, axes=(0, 0, 0)),
    # in-place, batched, scaled
    case(4, PE, R2C, (8, 16, 32), 2, 2, P2P, inplace=True),
    case(3, SL, C2C, (8, 8, 32), 3, 1, A2A, inplace=True, scale=(1.0, 1.0 / (8 * 8 * 32))),
    case(5, SL, R2C, (16, 8, 64), 5, 1, P2P, batch=3),
    case(6, PE, C2C, (16, 8, 16), 3, 2, P2P, batch=2, scale=(1 / math.sqrt(16 * 8 * 16),) * 2),
    case(4, ZY, None, (8, 16, 16), 4, 1, P2P, kinds=(DCT, DST, DCT), batch=2, inplace=True, scale=(0.5, 1.0 / (8 * 16 * 16 * 8))),
    case(2, PE, C2C, (16, 8, 64), 1, 2, P2P, scale=(1.0 / (16 * 8 * 64), 1.0)),
    case(3, PE, R2C, (8, 16, 64), 3, 1, A2A, d=2, inplace=True, batch=2, scale=(1.0 / (16 * 64), 1.0 / (16 * 64))),
    # f32
    case(8, PE, R2C, (16, 16, 128), 4, 2, P2P, prec=F32),
    case(5, SL, C2C, (16, 16, 128), 5, 1, P2P, STREAMS, prec=F32),
    case(3, SL, C2C, (48, 50, 45), 3, 1, A2A, prec=F32),
    case(6, PE, None, (16, 8, 32), 2, 3, P2P, prec=F32, kinds=MIXED),
    case(4, PE, C2C, (8, 16, 16), 2, 2, P2P, prec=F32, axes=(1, 0, 1), batch=2, inplace=True, scale=(0.25, 1.0)),
]


def both(c):
    p, _, d, env = c
    return [(p, 0, d, env), (p, 1, d, env)]


def case_id(c):
    p, inverse, d, env = c
    t = {C2C: "c2c", R2C: "r2c"}.get(p.transform, "r2r") if p.kinds is None else "r2r" + "".join("ctr"[k - 2] for k in p.kinds)
    parts = [f"P{p.P}", ["sl", "zy", "pe"][p.decomp] + f"{p.p1}x{p.p2}", t, "x".join(map(str, p.shape)),
             ["p2p", "a2a"][p.comm] + ["", "-str"][p.send], ["fwd", "inv"][inverse], f"d{d}", ["f32", "f64"][p.prec]]
    if p.axes is not None: parts.append("ax" + "".join(map(str, p.axes)))
    if p.fields > 1: parts.append(f"b{p.fields}")
    if p.inplace: parts.append("inpl")
    if p.scale is not None: parts.append("scaled")
    if env: parts.append("-".join(f"{k[5:].lower()}{v}" for k, v in env.items()))
    return "-".join(parts)


BASE = [case(P, decomp, t, shape, p1, p2, comm, send, inv) for P, decomp, t, shape, p1, p2, comm, send in CASES for inv in (0, 1)]
ALL = BASE + [c for e in EXTRA for c in both(e)]


@pytest.mark.gpu
@pytest.mark.parametrize("c", ALL, ids=case_id)
def test_replay(c, knobs):
    p, inverse, d, env = c
    knobs(env)
    check_case(p, inverse, d)


@pytest.mark.parametrize("c", [c for e in EXTRA for c in both(e)], ids=case_id)
def test_extra_cases_pass_the_cpu_replay(c, knobs):
    """every case added here passes its CPU replay as well: the overlapped schedules the C2C / R2C replay of
    test_schedule_emulation, in-place R2C / C2R (padded real rows) the replay of test_inplace, every other one the general
    replay of test_transform_axes"""
    p, inverse, d, env = c
    knobs(env)
    axes = p.axes or (1, 1, 1)
    if R.describe(p, 0, inverse, d)["overlapped"]:
        assert p.kinds is None and p.fields == 1 and not p.inplace and p.scale is None and axes == (1, 1, 1)
        assert run_case(p.P, p.decomp, p.transform, p.shape, p.p1, p.p2, p.comm, p.send, inverse, d, prec=p.prec) < 1e-12
    elif p.inplace and p.transform == R2C and p.kinds is None and axes == (1, 1, 1):
        scale = 1.0 if p.scale is None else p.scale[inverse]
        assert run_inplace(p.P, p.decomp, p.transform, p.shape, p.p1, p.p2, p.comm, p.send, inverse, d, p.fields, scale, p.prec) < 1e-12
    else:
        assert replay_cpu(p.P, p.decomp, p.transform, p.shape, p.p1, p.p2, axes, inverse, d, p.comm, p.send, p.kinds, p.fields, p.inplace,
                          p.scale, p.prec) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(8))
def test_random_replays(seed, knobs):
    """test_schedule_emulation's seeded random sweep (ranks 1-8, decompositions, grids, methods, directions, depths,
    precisions, layout and overlap knobs), here through the kernels"""
    rng = random.Random(1000 + seed)
    for i in range(10):
        rc, env = random_case(rng)
        p, inverse, d, _ = case(rc["P"], rc["decomp"], rc["transform"], rc["shape"], rc["p1"], rc["p2"], rc["comm_method"], rc["send_method"],
                                rc["inverse"], rc["d"], rc["prec"])
        knobs(env)
        check_case(p, inverse, d, seed=seed * 100 + i)


# ---- the checks are not vacuous ---------------------------------------------------------------------------------------------
NV = R.Plan(4, PE, (8, 12, 32), 2, 2)


def _first_pass(sched):
    return next(k for k, st in enumerate(sched["steps"]) if st["type"] == 0)


@pytest.mark.gpu
def test_a_skipped_pass_leaves_nan(knobs):
    knobs({})
    x, _ = global_input(NV, 0, 3, 0)
    outs = replay(NV, 0, 3, x, skip=(1, _first_pass(R.describe(NV, 1, 0, 3))))
    assert np.isnan(assemble(outs)).any()


@pytest.mark.gpu
def test_swapped_work_areas_change_the_result(knobs):
    knobs({})
    x, _ = global_input(NV, 0, 3, 0)
    good = assemble(replay(NV, 0, 3, x))

    def swap(r, work):  # rank 0's passes see ranks 0's and 1's areas exchanged
        return [work[1], work[0]] + work[2:] if r == 0 else work
    assert not same_bits(assemble(replay(NV, 0, 3, x, work_of=swap)), good)
    assert same_bits(good, one_rank(NV, 0, 3, x))


@pytest.mark.gpu
def test_one_bad_element_fails_the_max_bound(knobs):
    """50 u rms(ref) on one element exceeds 10 times the rel-L2 bound (sum log2 L = 2 here) though it barely moves the norm"""
    knobs({})
    p = R.Plan(4, PE, (8, 8, 4), 2, 2)
    got, ref = check_case(p, 0, 1)
    extra = np.zeros(ref.shape, dtype=ref.dtype)
    rms = float(np.sqrt(np.mean(np.abs(ref) ** 2)))
    extra[0, 3, 2, 1] = 50 * UNIT[p.prec] * rms
    rel, mx = error_check(geometry(p, 1), got, ref, extra)
    assert rel <= 3.0 and mx > 30.0


def _need(view, user, A0, A1, N, B, es):
    """bytes a buffer must hold for the view: offset of its base in the buffer (slots: in the rank's work area) + extent"""
    need = 0
    for base, ns, off in view_indices(view, A0, A1, N, B):
        start = base if user else work_offset(base)
        need = max(need, start + (int(off.max()) + 1) * es)
    return need


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["in", "out", "work"])
def test_short_buffers_are_refused(which, knobs):
    """a buffer one element short of a view's extent: DFFT_ERR_INVALID, and nothing is written"""
    knobs({})
    p = R.Plan(3, SL, (8, 16, 64), 3, 1, transform=R2C)
    with R.dry_plans(p, [0]) as (plan,):
        sc = R.schedule(p, plan, 0, 3)
        es = sc["esize"]
        work_bytes = sc["nslots"] * sc["slot_bytes"]
        _, _, bi, bo, _ = caller_buffers(p, sc, 0, 3, np.zeros((1,) + p.shape))
        for k, st in enumerate(sc["steps"]):
            if st["type"] != 0:
                continue
            N = st.get("n", 1 << st["log2n"])
            n_in, n_out = (N, N + 1) if st["kind"] == 2 else (N + 1, N) if st["kind"] == 3 else (N, N)
            need_in = _need(st["in"], st["in_user"], st["A0"], st["A1"], n_in, st["B"], es)
            need_out = _need(st["out"], st["out_user"], st["A0"], st["A1"], n_out, st["B"], es)
            sizes = dict(inp=bi.numel(), out=bo.numel(), work=work_bytes)
            if which == "in" and st["in_user"] == 1:
                sizes["inp"] = need_in
            elif which == "out" and st["out_user"] == 2:
                sizes["out"] = need_out
            elif which == "work" and st["in_user"] == 0 and st["out_user"] == 0:
                sizes["work"] = max(need_in, need_out)
            else:
                continue
            key = {"in": "inp"}.get(which, which)
            work = [nan_buffer(work_bytes) for _ in range(3)]
            torch.cuda.synchronize()
            before = [t_.clone() for t_ in work + [bi, bo]]
            run = lambda sz: run_step(plan, 0, 3, 0, k, work, sz["work"], bo, sz["out"], bi, sz["inp"])
            assert run(dict(sizes, **{key: sizes[key] - es})) == ERR_INVALID
            torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(before, work + [bi, bo])), "a refused step wrote"
            assert run(sizes) == 0  # the exact extent is enough
            return
        pytest.fail("no step with such a view")


@pytest.mark.gpu
def test_hook_refuses_other_steps_and_plans(knobs):
    """rendezvous and all-to-all steps, steps and fields out of range, and plans that are not geometry-only"""
    knobs({})
    for p, t in ((R.Plan(4, SL, (8, 8, 32), 4, 1, comm=A2A), 2), (NV, 1)):
        with R.dry_plans(p, [0]) as (plan,):
            sc = R.schedule(p, plan, 0, 3)
            wb = sc["nslots"] * sc["slot_bytes"]
            work = [nan_buffer(wb) for _ in range(4)]
            b = nan_buffer(1 << 16)
            k = next(k for k, st in enumerate(sc["steps"]) if st["type"] == t)
            assert run_step(plan, 0, 3, 0, k, work, wb, b, b.numel(), b, b.numel()) == ERR_UNSUPPORTED
            assert run_step(plan, 0, 3, 0, len(sc["steps"]), work, wb, b, b.numel(), b, b.numel()) == ERR_INVALID
            assert run_step(plan, 0, 3, 1, _first_pass(sc), work, wb, b, b.numel(), b, b.numel()) == ERR_INVALID
    comm = C.c_void_p()
    check(lib().dfft_comm_create(0, 1, None, torch.cuda.current_device(), C.byref(comm)))
    plan = one_rank_plan(NV, comm)
    try:
        assert run_step(plan, 0, 3, 0, 0, work, wb, b, b.numel(), b, b.numel()) == -4  # DFFT_ERR_STATE
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(comm)
