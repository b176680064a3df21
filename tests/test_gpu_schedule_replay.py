"""Replays multi-rank schedules on one GPU with the real pass kernels.

The CPU replays (test_schedule_emulation and the family replays) check the data movement of every rank's step list with
numpy in place of the kernels.  Here the same step lists run on one H100 through dfft_debug_run_step: every rank gets its
own work area and user buffers, the ranks run in lock step (pass steps through the hook, all-to-all steps as device copies,
rendezvous as no-ops), so the multi-rank kernel paths execute — multi-segment views, stores into other ranks' slots with the
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

import numpy as np
import pytest
import torch

import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from step_replay import view_indices
from test_inplace import run_inplace
from test_schedule_emulation import CASES, KNOBS, random_case, run_case
from test_transform_axes import describe_raw, fwd_ref, inv_ref, run as replay_cpu, set_axes

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
C2C, R2C, DCT, DST, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.DST, dfft.R2HC
F32, F64 = dfft.F32, dfft.F64
ERR_INVALID, ERR_UNSUPPORTED = -1, -5
SLOT_SHIFT = 44  # synthetic slot address of rank r: ((r+1) << 44) + offset
UNIT = {F64: 2.0 ** -53, F32: 2.0 ** -24}
WORST = {}  # (family, precision) -> worst measured (rel-L2, max) error in units of u sqrt(sum log2 L)


def spec(P, decomp, transform, shape, p1, p2, comm=P2P, send=SYNC, inverse=0, d=3, prec=F64, kinds=None, axes=(1, 1, 1), batch=1,
         inplace=False, scale=None, env=None):
    return dict(P=P, decomp=decomp, transform=transform, shape=tuple(shape), p1=p1, p2=p2, comm=comm, send=send, inverse=inverse, d=d, prec=prec,
                kinds=kinds, axes=tuple(axes), batch=batch, inplace=inplace, scale=scale, env=env or {})


# ---- plans ------------------------------------------------------------------------------------------------------------------
def make_plan(comm, s, p1, p2, allocate):
    cfg = _lib.dfft_config(1, 0, s["comm"], s["send"], None, s["comm"], s["send"])
    plan = C.c_void_p()
    nx, ny, nz = s["shape"]
    if s["kinds"] is not None:
        rc = lib().dfft_plan_create_r2r(comm, C.byref(cfg), s["decomp"], s["prec"], (C.c_int * 3)(*s["kinds"]), nx, ny, nz, p1, p2, s["batch"],
                                        int(s["inplace"]), allocate, C.byref(plan))
    else:
        fn = lib().dfft_plan_create_inplace if s["inplace"] else lib().dfft_plan_create_batched
        rc = fn(comm, C.byref(cfg), s["decomp"], s["prec"], s["transform"], nx, ny, nz, p1, p2, s["batch"], allocate, C.byref(plan))
    check(rc)
    if s["axes"] != (1, 1, 1):
        check(set_axes(plan, s["axes"]))
    if s["scale"] is not None:
        check(lib().dfft_plan_set_scale(plan, *s["scale"]))
    return plan


class DryPlans:
    """the geometry-only plans of all P ranks with their step lists"""

    def __init__(self, s):
        import json
        self.comms, self.plans, self.scheds = [], [], []
        for r in range(s["P"]):
            c = C.c_void_p()
            check(lib().dfft_comm_create_dry(r, s["P"], C.byref(c)))
            self.comms.append(c)
            self.plans.append(make_plan(c, s, s["p1"], s["p2"], 1))
            sc = json.loads(describe_raw(self.plans[-1], s["inverse"], s["d"]))
            sc["domain_bytes"] = lib().dfft_get_domain_size(self.plans[-1])
            self.scheds.append(sc)

    def close(self):
        for plan, c in zip(self.plans, self.comms):
            lib().dfft_plan_destroy(plan)
            lib().dfft_comm_destroy(c)


# ---- buffers: the layouts of test_transform_axes.run, in device memory ------------------------------------------------------
def dtypes(s, real):
    f64 = s["prec"] == F64
    if real:
        return (np.float64, torch.float64) if f64 else (np.float32, torch.float32)
    return (np.complex128, torch.complex128) if f64 else (np.complex64, torch.complex64)


class Side:
    """one rank's caller buffer on one side (in / out) of an exec: its blocks of the global array, field by field"""

    def __init__(self, s, rank, p1, p2, which, real, r2c_real, es, domain_bytes):
        nx, ny, nz = s["shape"]
        lay_t = DCT if s["kinds"] is not None else s["transform"]
        self.size, self.start = dfft.layout(s["decomp"], lay_t, nx, ny, nz, p1, p2, rank, which)
        self.real, self.r2c_real, self.es = real, r2c_real, es
        self.nz = nz
        # R2C: the real side in complex units; in-place plans: rows padded to Nz/2+1 complex units, fields domain bytes apart
        self.padded = r2c_real and s["inplace"]
        row = (nz // 2 + 1) if self.padded else (self.size[2] // 2 if r2c_real else self.size[2])
        self.elems = self.size[0] * self.size[1] * row
        self.field = domain_bytes // es if s["inplace"] else self.elems
        self.nbytes = max(s["batch"] * max(self.field, self.elems), 1) * es
        self.npdt, self.tdt = dtypes(s, real)

    def view(self, buf, f):
        off = f * self.field * self.es
        t = buf[off:off + self.elems * self.es].view(self.tdt)
        if self.padded:
            return t.view(self.size[0], self.size[1], -1)[:, :, :self.nz]
        return t.view(*self.size)

    def put(self, buf, f, block):
        self.view(buf, f).copy_(torch.from_numpy(np.ascontiguousarray(block.astype(self.npdt))))

    def get(self, buf, f):
        return self.view(buf, f).cpu().numpy()


def sides(s, P, p1, p2, domain_bytes, es):
    """(in side, out side) per rank"""
    real = s["kinds"] is not None
    r2c = s["transform"] == R2C and not real
    src_w, dst_w = (s["d"], 0) if s["inverse"] else (0, s["d"])
    out = []
    for r in range(P):
        i = Side(s, r, p1, p2, src_w, real or (r2c and not s["inverse"]), r2c and not s["inverse"], es, domain_bytes[r])
        o = Side(s, r, p1, p2, dst_w, real or (r2c and s["inverse"]), r2c and bool(s["inverse"]), es, domain_bytes[r])
        out.append((i, o))
    return out


def nan_buffer(nbytes):
    return torch.full((nbytes,), 0xFF, dtype=torch.uint8, device="cuda")  # 0xFF..: NaN in f32 and f64


def block(a, start, size):
    return a[start[0]:start[0] + size[0], start[1]:start[1] + size[1], start[2]:start[2] + size[2]]


# ---- inputs and the long-double reference ----------------------------------------------------------------------------------
def global_input(s, seed):
    """(input in the plan's precision, the same values in long double) of shape (batch, ...) — zero-mean normal; an inverse
    R2C input is the forward transform of real normal data, so that it is the spectrum of a real array"""
    rng = np.random.default_rng(seed)
    nx, ny, nz = s["shape"]
    b = s["batch"]
    real = s["kinds"] is not None
    cplx_dt, real_dt = dtypes(s, False)[0], dtypes(s, True)[0]
    if s["inverse"] and s["transform"] == R2C and not real:
        x = rng.standard_normal((b, nx, ny, nz)).astype(np.longdouble)
        X = np.stack([fwd_ref(x[f], R2C, None, s["axes"], s["d"]) for f in range(b)]).astype(cplx_dt)
        return X, X.astype(np.clongdouble)
    shape = (b, nx, ny, nz)
    if real or (s["transform"] == R2C and not s["inverse"]):
        x = rng.standard_normal(shape).astype(real_dt)
        return x, x.astype(np.longdouble)
    x = (rng.standard_normal(shape) + 1j * rng.standard_normal(shape)).astype(cplx_dt)
    return x, x.astype(np.clongdouble)


def reference(s, x_ld):
    kinds = s["kinds"]
    t = s["transform"] if kinds is None else None
    if s["inverse"]:
        y = np.stack([inv_ref(x_ld[f], t, kinds, s["axes"], s["d"], s["shape"][2]) for f in range(s["batch"])])
    else:
        y = np.stack([fwd_ref(x_ld[f], t, kinds, s["axes"], s["d"]) for f in range(s["batch"])])
    sc = 1.0 if s["scale"] is None else s["scale"][1 if s["inverse"] else 0]
    if s["prec"] == F32:
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


def family(s):
    if any(not s["axes"][a] for a in (2, 1, 0)[:s["d"]]):
        return "copy"
    if s["kinds"] is not None:
        return "R2R"
    if any(s["shape"][a] & (s["shape"][a] - 1) for a in (2, 1, 0)[:s["d"]] if s["axes"][a]):
        return "Bluestein"
    return "R2C/C2R" if s["transform"] == R2C else "C2C"


def error_check(s, got, want, extra=None):
    """check 2; returns (rel-L2, max) in units of u sqrt(sum log2 L)"""
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
def run_step(plan, s, field, step, work, work_bytes, out, out_bytes, inp, in_bytes):
    ptrs = (C.c_void_p * len(work))(*[w.data_ptr() for w in work])
    return lib().dfft_debug_run_step(plan, s["inverse"], s["d"], field, step, ptrs, work_bytes, out.data_ptr(), out_bytes, inp.data_ptr(), in_bytes,
                                     torch.cuda.current_stream().cuda_stream)


def replay(s, dry, x, descending=False, skip=None, work_of=None):
    """every rank's steps in lock step on this GPU; returns (per-rank input buffers, output buffers, sides).
    skip = (rank, item): a pass not run; work_of(rank, work): the work areas rank's passes see"""
    P = s["P"]
    scheds = dry.scheds
    es = scheds[0]["esize"]
    nslots, slot_bytes = scheds[0]["nslots"], scheds[0]["slot_bytes"]
    assert all(sc["nslots"] == nslots and sc["slot_bytes"] == slot_bytes for sc in scheds)
    work_bytes = nslots * slot_bytes
    work = [nan_buffer(work_bytes) for _ in range(P)]
    sd = sides(s, P, s["p1"], s["p2"], [sc["domain_bytes"] for sc in scheds], es)
    ins, outs = [], []
    for r in range(P):
        si, so = sd[r]
        bi = nan_buffer(max(si.nbytes, so.nbytes) if s["inplace"] else si.nbytes)
        for f in range(s["batch"]):
            si.put(bi, f, block(x[f], si.start, si.size))
        ins.append(bi)
        outs.append(bi if s["inplace"] else nan_buffer(so.nbytes))
    items = len(scheds[0]["steps"])
    assert all(len(sc["steps"]) == items for sc in scheds)
    per = items // s["batch"]
    for k in range(items):
        for r in (reversed(range(P)) if descending else range(P)):
            st = scheds[r]["steps"][k]
            if st["type"] == 1:
                continue  # rendezvous: the lock step orders everything
            if st["type"] == 2:  # all-to-all-v between staging slots
                sb = scheds[r]["slots"][st["send_slot"]][r] - ((r + 1) << SLOT_SHIFT)
                for peer in st["peers"]:
                    q = peer["rank"]
                    rb = scheds[q]["slots"][st["recv_slot"]][q] - ((q + 1) << SLOT_SHIFT)
                    mine = [pp for pp in scheds[q]["steps"][k]["peers"] if pp["rank"] == r][0]
                    n = peer["scount"] * es
                    so_, ro = sb + peer["soff"] * es, rb + mine["roff"] * es
                    work[q][ro:ro + n].copy_(work[r][so_:so_ + n])
                continue
            if skip == (r, k):
                continue
            w = work_of(r, work) if work_of else work
            rc = run_step(dry.plans[r], s, k // per, k % per, w, work_bytes, outs[r], outs[r].numel(), ins[r], ins[r].numel())
            assert rc == 0, f"rank {r} step {k} ({st['label']}): {(lib().dfft_last_error_string() or b'').decode()}"
    torch.cuda.synchronize()
    return ins, outs, sd


def assemble(s, sd, bufs, which):
    """the global array (batch, ...) from every rank's blocks on one side (0 in, 1 out)"""
    nx, ny, nz = s["shape"]
    first = sd[0][which]
    zext = max(sd[r][which].start[2] + sd[r][which].size[2] for r in range(len(sd)))
    g = np.zeros((s["batch"], nx, ny, zext), dtype=first.npdt)
    for r, sides_r in enumerate(sd):
        side = sides_r[which]
        for f in range(s["batch"]):
            block(g[f], side.start, side.size)[...] = side.get(bufs[r], f)
    return g


def one_rank(s, x):
    """the real one-rank plan of the same transform on the whole grid: its output (batch, ...)"""
    comm = C.c_void_p()
    check(lib().dfft_comm_create(0, 1, None, torch.cuda.current_device(), C.byref(comm)))
    plan = make_plan(comm, s, 1, 1, 1)
    try:
        es = (8 if s["kinds"] is not None else 16) // (1 if s["prec"] == F64 else 2)  # bytes per view element
        (si, so), = sides(s, 1, 1, 1, [lib().dfft_get_domain_size(plan)], es)
        bi = nan_buffer(max(si.nbytes, so.nbytes) if s["inplace"] else si.nbytes)
        for f in range(s["batch"]):
            si.put(bi, f, x[f])
        bo = bi if s["inplace"] else nan_buffer(so.nbytes)
        torch.cuda.synchronize()
        direction = 1 if s["inverse"] else -1
        if s["kinds"] is not None:
            check(lib().dfft_exec_r2r_partial(plan, bo.data_ptr(), bi.data_ptr(), direction, s["d"]))
        elif s["transform"] == C2C:
            check(lib().dfft_exec_c2c_partial(plan, bo.data_ptr(), bi.data_ptr(), direction, s["d"]))
        elif s["inverse"]:
            check(lib().dfft_exec_c2r_partial(plan, bo.data_ptr(), bi.data_ptr(), s["d"]))
        else:
            check(lib().dfft_exec_r2c_partial(plan, bo.data_ptr(), bi.data_ptr(), s["d"]))
        return np.stack([so.get(bo, f) for f in range(s["batch"])])
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(comm)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def check_case(s, seed=0):
    dry = DryPlans(s)
    try:
        x, x_ld = global_input(s, seed)
        ins, outs, sd = replay(s, dry, x)
        got = assemble(s, sd, outs, 1)
        # 3: no element left unwritten, the inputs intact
        assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements were never written"
        if not s["inplace"]:
            for f in range(s["batch"]):
                for r, (si, _) in enumerate(sd):
                    assert same_bits(si.get(ins[r], f), block(x[f], si.start, si.size).astype(si.npdt)), f"rank {r} field {f}: input changed"
        # the ranks of each step in the other order: the same bits
        _, outs2, _ = replay(s, dry, x, descending=True)
        assert same_bits(assemble(s, sd, outs2, 1), got), "the result depends on the order of the ranks within a step"
    finally:
        dry.close()
    # 1: the one-rank plan on the whole grid
    if s["kinds"] is None:
        want1 = one_rank(s, x)
        assert same_bits(got, want1), f"differs from the one-rank plan at {np.argwhere(got != want1)[:8].tolist()}"
    # else: R2R passes transform lines in pairs (two real lines as one complex line), and which lines pair up follows the
    # rank-local line and column counts, so the rounding differs from the one-rank plan's; check 2 covers them
    # 2: the long-double reference
    ref = reference(s, x_ld)
    rel, mx = error_check(s, got, ref)
    key = (family(s), "f64" if s["prec"] == F64 else "f32")
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
    spec(2, SL, C2C, (8, 32, 64), 2, 1, A2A),
    spec(3, SL, R2C, (16, 16, 64), 3, 1, P2P, STREAMS),
    spec(5, SL, C2C, (16, 16, 128), 5, 1, P2P),
    spec(5, ZY, R2C, (16, 8, 64), 5, 1, A2A),
    spec(7, ZY, C2C, (16, 8, 64), 7, 1, P2P),
    spec(6, PE, C2C, (16, 16, 32), 3, 2, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    spec(6, PE, R2C, (8, 16, 64), 2, 3, A2A),
    spec(7, PE, C2C, (16, 8, 32), 7, 1, P2P),  # P2 = 1
    spec(7, PE, R2C, (8, 16, 64), 1, 7, P2P),  # P1 = 1
    spec(8, PE, R2C, (16, 8, 128), 4, 2, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    spec(8, SL, C2C, (32, 16, 64), 8, 1, P2P, STREAMS),
    spec(3, PE, C2C, (16, 16, 32), 3, 1, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    spec(5, SL, R2C, (16, 32, 128), 5, 1, P2P, STREAMS, env={"DFFT_XCHG_CTAS": "32"}),
    # partial d
    spec(6, PE, R2C, (8, 16, 64), 3, 2, P2P, d=1),
    spec(6, PE, C2C, (16, 8, 64), 2, 3, A2A, d=2),
    # long axes: wide tiles and the TMA-fed kernel on single-segment local passes
    spec(2, SL, C2C, (8, 16, 8192), 2, 1, P2P),
    spec(4, PE, R2C, (16, 8, 4096), 2, 2, P2P),
    spec(3, SL, C2C, (8, 1024, 32), 3, 1, A2A),
    spec(4, ZY, C2C, (2048, 8, 16), 4, 1, P2P),
    spec(8, PE, C2C, (1024, 16, 32), 2, 4, P2P, STREAMS, env={"DFFT_PENCIL_OVERLAP": "2"}),
    # R2C with odd Nzc tails
    spec(3, SL, R2C, (8, 16, 256), 3, 1, P2P),  # Nzc = 129
    spec(5, PE, R2C, (16, 16, 32), 1, 5, P2P),  # Nzc = 17 over 5
    # Bluestein lengths
    spec(3, SL, C2C, (96, 100, 90), 3, 1, P2P),
    spec(4, PE, C2C, (12, 30, 27), 2, 2, A2A),
    spec(5, ZY, C2C, (20, 24, 45), 5, 1, P2P),
    # DCT, DST and mixed kinds with odd rank-local counts
    spec(3, SL, None, (16, 8, 32), 3, 1, P2P, kinds=(DCT, DCT, DCT)),
    spec(5, PE, None, (16, 16, 16), 1, 5, A2A, kinds=(DST, DST, DST)),
    spec(6, PE, None, (8, 16, 32), 3, 2, P2P, kinds=MIXED),
    spec(7, ZY, None, (16, 8, 32), 7, 1, P2P, kinds=(DCT, R2HC, DST)),
    # kept axes (copy passes)
    spec(4, PE, C2C, (8, 16, 32), 2, 2, P2P, axes=(0, 1, 1)),
    spec(3, SL, R2C, (8, 8, 32), 3, 1, A2A, axes=(1, 0, 1)),
    spec(5, ZY, None, (16, 8, 16), 5, 1, P2P, kinds=MIXED, axes=(1, 1, 0)),
    spec(6, PE, C2C, (8, 16, 16), 3, 2, P2P, axes=(0, 0, 0)),
    # in-place, batched, scaled
    spec(4, PE, R2C, (8, 16, 32), 2, 2, P2P, inplace=True),
    spec(3, SL, C2C, (8, 8, 32), 3, 1, A2A, inplace=True, scale=(1.0, 1.0 / (8 * 8 * 32))),
    spec(5, SL, R2C, (16, 8, 64), 5, 1, P2P, batch=3),
    spec(6, PE, C2C, (16, 8, 16), 3, 2, P2P, batch=2, scale=(1 / math.sqrt(16 * 8 * 16),) * 2),
    spec(4, ZY, None, (8, 16, 16), 4, 1, P2P, kinds=(DCT, DST, DCT), batch=2, inplace=True, scale=(0.5, 1.0 / (8 * 16 * 16 * 8))),
    spec(2, PE, C2C, (16, 8, 64), 1, 2, P2P, scale=(1.0 / (16 * 8 * 64), 1.0)),
    spec(3, PE, R2C, (8, 16, 64), 3, 1, A2A, d=2, inplace=True, batch=2, scale=(1.0 / (16 * 64), 1.0 / (16 * 64))),
    # f32
    spec(8, PE, R2C, (16, 16, 128), 4, 2, P2P, prec=F32),
    spec(5, SL, C2C, (16, 16, 128), 5, 1, P2P, STREAMS, prec=F32),
    spec(3, SL, C2C, (48, 50, 45), 3, 1, A2A, prec=F32),
    spec(6, PE, None, (16, 8, 32), 2, 3, P2P, prec=F32, kinds=MIXED),
    spec(4, PE, C2C, (8, 16, 16), 2, 2, P2P, prec=F32, axes=(1, 0, 1), batch=2, inplace=True, scale=(0.25, 1.0)),
]


def both(s):
    return [dict(s, inverse=0), dict(s, inverse=1)]


def case_id(s):
    t = {C2C: "c2c", R2C: "r2c"}.get(s["transform"], "r2r") if s["kinds"] is None else "r2r" + "".join("ctr"[k - 2] for k in s["kinds"])
    parts = [f"P{s['P']}", ["sl", "zy", "pe"][s["decomp"]] + f"{s['p1']}x{s['p2']}", t, "x".join(map(str, s["shape"])),
             ["p2p", "a2a"][s["comm"]] + ["", "-str"][s["send"]], ["fwd", "inv"][s["inverse"]], f"d{s['d']}", ["f32", "f64"][s["prec"]]]
    if s["axes"] != (1, 1, 1): parts.append("ax" + "".join(map(str, s["axes"])))
    if s["batch"] > 1: parts.append(f"b{s['batch']}")
    if s["inplace"]: parts.append("inpl")
    if s["scale"] is not None: parts.append("scaled")
    if s["env"]: parts.append("-".join(f"{k[5:].lower()}{v}" for k, v in s["env"].items()))
    return "-".join(parts)


BASE = [spec(P, decomp, t, shape, p1, p2, comm, send, inv) for P, decomp, t, shape, p1, p2, comm, send in CASES for inv in (0, 1)]
ALL = BASE + [c for s in EXTRA for c in both(s)]


@pytest.mark.gpu
@pytest.mark.parametrize("s", ALL, ids=case_id)
def test_replay(s, knobs):
    knobs(s["env"])
    check_case(s)


@pytest.mark.parametrize("s", [c for s in EXTRA for c in both(s)], ids=case_id)
def test_extra_cases_pass_the_cpu_replay(s, knobs):
    """every case added here passes its CPU replay as well: the overlapped schedules the C2C / R2C replay of
    test_schedule_emulation, in-place R2C / C2R (padded real rows) the replay of test_inplace, every other one the general
    replay of test_transform_axes"""
    knobs(s["env"])
    dry = DryPlans(s)
    overlapped = dry.scheds[0]["overlapped"]
    dry.close()
    if overlapped:
        assert s["kinds"] is None and s["batch"] == 1 and not s["inplace"] and s["scale"] is None and s["axes"] == (1, 1, 1)
        assert run_case(s["P"], s["decomp"], s["transform"], s["shape"], s["p1"], s["p2"], s["comm"], s["send"], s["inverse"], s["d"],
                        prec=s["prec"]) < 1e-12
    elif s["inplace"] and s["transform"] == R2C and s["kinds"] is None and s["axes"] == (1, 1, 1):
        scale = 1.0 if s["scale"] is None else s["scale"][s["inverse"]]
        assert run_inplace(s["P"], s["decomp"], s["transform"], s["shape"], s["p1"], s["p2"], s["comm"], s["send"], s["inverse"], s["d"], s["batch"],
                           scale, s["prec"]) < 1e-12
    else:
        assert replay_cpu(s["P"], s["decomp"], s["transform"], s["shape"], s["p1"], s["p2"], s["axes"], s["inverse"], s["d"], s["comm"], s["send"],
                          s["kinds"], s["batch"], s["inplace"], s["scale"], s["prec"]) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(8))
def test_random_replays(seed, knobs):
    """test_schedule_emulation's seeded random sweep (ranks 1-8, decompositions, grids, methods, directions, depths,
    precisions, layout and overlap knobs), here through the kernels"""
    rng = random.Random(1000 + seed)
    for i in range(10):
        case, env = random_case(rng)
        s = spec(case["P"], case["decomp"], case["transform"], case["shape"], case["p1"], case["p2"], case["comm_method"], case["send_method"],
                 case["inverse"], case["d"], case["prec"], env=env)
        knobs(env)
        check_case(s, seed=seed * 100 + i)


# ---- the checks are not vacuous ---------------------------------------------------------------------------------------------
NV = spec(4, PE, C2C, (8, 12, 32), 2, 2, P2P)


def _first_pass(sched):
    return next(k for k, st in enumerate(sched["steps"]) if st["type"] == 0)


@pytest.mark.gpu
def test_a_skipped_pass_leaves_nan(knobs):
    knobs({})
    dry = DryPlans(NV)
    try:
        x, _ = global_input(NV, 0)
        _, outs, sd = replay(NV, dry, x, skip=(1, _first_pass(dry.scheds[1])))
        assert np.isnan(assemble(NV, sd, outs, 1)).any()
    finally:
        dry.close()


@pytest.mark.gpu
def test_swapped_work_areas_change_the_result(knobs):
    knobs({})
    dry = DryPlans(NV)
    try:
        x, _ = global_input(NV, 0)
        _, outs, sd = replay(NV, dry, x)
        good = assemble(NV, sd, outs, 1)

        def swap(r, work):  # rank 0's passes see ranks 0's and 1's areas exchanged
            return [work[1], work[0]] + work[2:] if r == 0 else work
        _, outs, _ = replay(NV, dry, x, work_of=swap)
        assert not same_bits(assemble(NV, sd, outs, 1), good)
    finally:
        dry.close()
    assert same_bits(good, one_rank(NV, x))


@pytest.mark.gpu
def test_one_bad_element_fails_the_max_bound(knobs):
    """50 u rms(ref) on one element exceeds 10 times the rel-L2 bound (sum log2 L = 2 here) though it barely moves the norm"""
    knobs({})
    s = spec(4, PE, C2C, (8, 8, 4), 2, 2, P2P, d=1)
    got, ref = check_case(s)
    extra = np.zeros(ref.shape, dtype=ref.dtype)
    rms = float(np.sqrt(np.mean(np.abs(ref) ** 2)))
    extra[0, 3, 2, 1] = 50 * UNIT[s["prec"]] * rms
    rel, mx = error_check(s, got, ref, extra)
    assert rel <= 3.0 and mx > 30.0


def _need(view, user, A0, A1, N, B, es):
    """bytes a buffer must hold for the view: offset of its base in the buffer (slots: in the rank's work area) + extent"""
    need = 0
    for base, ns, off in view_indices(view, A0, A1, N, B):
        start = base if user else base - ((base >> SLOT_SHIFT) << SLOT_SHIFT)
        need = max(need, start + (int(off.max()) + 1) * es)
    return need


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["in", "out", "work"])
def test_short_buffers_are_refused(which, knobs):
    """a buffer one element short of a view's extent: DFFT_ERR_INVALID, and nothing is written"""
    knobs({})
    s = spec(3, SL, R2C, (8, 16, 64), 3, 1, P2P)
    dry = DryPlans(s)
    try:
        sc = dry.scheds[0]
        es = sc["esize"]
        si, so = sides(s, 3, 3, 1, [q["domain_bytes"] for q in dry.scheds], es)[0]
        work_bytes = sc["nslots"] * sc["slot_bytes"]
        for k, st in enumerate(sc["steps"]):
            if st["type"] != 0:
                continue
            N = st.get("n", 1 << st["log2n"])
            n_in, n_out = (N, N + 1) if st["kind"] == 2 else (N + 1, N) if st["kind"] == 3 else (N, N)
            need_in = _need(st["in"], st["in_user"], st["A0"], st["A1"], n_in, st["B"], es)
            need_out = _need(st["out"], st["out_user"], st["A0"], st["A1"], n_out, st["B"], es)
            sizes = dict(inp=si.nbytes, out=so.nbytes, work=work_bytes)
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
            bi, bo = nan_buffer(si.nbytes), nan_buffer(so.nbytes)
            si.put(bi, 0, np.zeros(si.size))
            torch.cuda.synchronize()
            before = [t_.clone() for t_ in work + [bi, bo]]
            run = lambda sz: run_step(dry.plans[0], s, 0, k, work, sz["work"], bo, sz["out"], bi, sz["inp"])
            assert run(dict(sizes, **{key: sizes[key] - es})) == ERR_INVALID
            torch.cuda.synchronize()
            assert all(torch.equal(a, b) for a, b in zip(before, work + [bi, bo])), "a refused step wrote"
            assert run(sizes) == 0  # the exact extent is enough
            return
        pytest.fail("no step with such a view")
    finally:
        dry.close()


@pytest.mark.gpu
def test_hook_refuses_other_steps_and_plans(knobs):
    """rendezvous and all-to-all steps, steps and fields out of range, and plans that are not geometry-only"""
    knobs({})
    for s, t in ((spec(4, SL, C2C, (8, 8, 32), 4, 1, A2A), 2), (NV, 1)):
        dry = DryPlans(s)
        try:
            sc = dry.scheds[0]
            wb = sc["nslots"] * sc["slot_bytes"]
            work = [nan_buffer(wb) for _ in range(4)]
            b = nan_buffer(1 << 16)
            k = next(k for k, st in enumerate(sc["steps"]) if st["type"] == t)
            assert run_step(dry.plans[0], s, 0, k, work, wb, b, b.numel(), b, b.numel()) == ERR_UNSUPPORTED
            assert run_step(dry.plans[0], s, 0, len(sc["steps"]), work, wb, b, b.numel(), b, b.numel()) == ERR_INVALID
            assert run_step(dry.plans[0], s, 1, _first_pass(sc), work, wb, b, b.numel(), b, b.numel()) == ERR_INVALID
        finally:
            dry.close()
    comm = C.c_void_p()
    check(lib().dfft_comm_create(0, 1, None, torch.cuda.current_device(), C.byref(comm)))
    plan = make_plan(comm, dict(NV, P=1), 1, 1, 1)
    try:
        assert run_step(plan, NV, 0, 0, work, wb, b, b.numel(), b, b.numel()) == -4  # DFFT_ERR_STATE
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(comm)
