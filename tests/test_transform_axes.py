"""Plans with untransformed (kept) axes (dfft_plan_set_transform_axes) without a GPU.

- Validation of the setter and getter, DFFT_ERR_STATE once a schedule exists, and byte-identical descriptions of plans
  whose axes are all transformed, with and without a {1, 1, 1} setter call.
- Lock-step replays of every rank's step list (test_schedule_emulation's Ordering / view_indices): numpy / scipy per
  pass, a plain element copy for the copy passes (kinds 6 / 7), checked against the transform of only the transformed
  axes among the first d stages: all 8 masks for C2C and for mixed-kind R2R, the 4 R2C masks that transform z, 1-8 ranks,
  slab, Z_Then_YX and pencil, Peer2Peer and All2All, Streams (sequential), partial d, uneven splits, blocked tails,
  Bluestein lengths, batches, in-place plans and scales (each output value scaled exactly once).
- The elision rules on the step lists (DESIGN.md section 3.12), and a broken copy step that the replay rejects."""
import ctypes as C
import itertools
import json

import numpy as np
import pytest

import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from test_r2r import CASES as R2R_CASES
from test_r2r_mixed import r2r_1d
from test_schedule_emulation import Memory, Ordering, view_indices

SL, ZY, PE = dfft.SLAB_ZY_THEN_X, dfft.SLAB_Z_THEN_YX, dfft.PENCIL
P2P, A2A = 0, 1
SYNC, STREAMS = 0, 1
USER_IN, USER_OUT = 1 << 60, 1 << 61
C2C, R2C, DCT, DST, R2HC = dfft.C2C, dfft.R2C, dfft.DCT, dfft.DST, dfft.R2HC
ERR_INVALID, ERR_STATE = -1, -4  # include/dfft.h
MASKS = list(itertools.product((0, 1), repeat=3))  # (x, y, z)
R2C_MASKS = [m for m in MASKS if m[2]]
MIXED = (R2HC, DST, DCT)
KIND = {"dct": DCT, "dst": DST, "r2hc": R2HC}


def mask_id(m):
    return "".join("t" if a else "k" for a in m)


# ---- plans ------------------------------------------------------------------------------------------------------------
def create(rank, P, decomp, transform, shape, p1, p2, comm=P2P, send=SYNC, batch=1, inplace=False, prec=dfft.F64, kinds=None):
    """dry plan: (rc, comm, plan); kinds: a per-axis real-to-real plan"""
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(rank, P, C.byref(c)))
    cfg = _lib.dfft_config(1, 0, comm, send, None, comm, send)
    plan = C.c_void_p()
    if kinds is not None:
        rc = lib().dfft_plan_create_r2r(c, C.byref(cfg), decomp, prec, (C.c_int * 3)(*kinds), *shape, p1, p2, batch, 1 if inplace else 0, 1,
                                        C.byref(plan))
    else:
        fn = lib().dfft_plan_create_inplace if inplace else lib().dfft_plan_create_batched
        rc = fn(c, C.byref(cfg), decomp, prec, transform, *shape, p1, p2, batch, 1, C.byref(plan))
    assert rc == 0, (lib().dfft_last_error_string() or b"").decode()
    return c, plan


def destroy(c, plan):
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)


def set_axes(plan, axes):
    return lib().dfft_plan_set_transform_axes(plan, None if axes is None else (C.c_int * 3)(*axes))


def describe_raw(plan, inverse, d):
    need = C.c_size_t()
    check(lib().dfft_plan_describe(plan, inverse, d, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib().dfft_plan_describe(plan, inverse, d, buf, need.value, C.byref(need)))
    return buf.value.decode()


def describe(rank, P, decomp, transform, shape, p1, p2, axes, inverse, d, comm=P2P, send=SYNC, batch=1, inplace=False, scale=None,
             prec=dfft.F64, kinds=None):
    c, plan = create(rank, P, decomp, transform, shape, p1, p2, comm, send, batch, inplace, prec, kinds)
    if axes is not None:
        assert set_axes(plan, axes) == 0, (lib().dfft_last_error_string() or b"").decode()
    if scale is not None:
        assert lib().dfft_plan_set_scale(plan, *scale) == 0
    sc = json.loads(describe_raw(plan, inverse, d))
    sc["domain_bytes"] = lib().dfft_get_domain_size(plan)
    destroy(c, plan)
    return sc


# ---- validation ---------------------------------------------------------------------------------------------------------
def test_validation_and_default():
    t = (C.c_int * 3)()
    c, plan = create(0, 1, SL, C2C, (8, 16, 32), 1, 1)
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 1, 1)
    assert lib().dfft_plan_get_transform_axes(None, t) == ERR_INVALID
    assert lib().dfft_plan_get_transform_axes(plan, None) == ERR_INVALID
    assert set_axes(None, (1, 1, 0)) == ERR_INVALID
    assert set_axes(plan, None) == ERR_INVALID
    for bad in ((2, 1, 1), (1, -1, 1), (1, 1, 3), (0, 0, 7)):
        assert set_axes(plan, bad) == ERR_INVALID, bad
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 1, 1)  # refused calls change nothing
    assert set_axes(plan, (0, 1, 1)) == 0
    assert set_axes(plan, (1, 0, 0)) == 0  # may be set again until a schedule exists
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 0, 0)
    describe_raw(plan, 0, 3)
    assert set_axes(plan, (1, 1, 1)) == ERR_STATE
    check(lib().dfft_plan_get_transform_axes(plan, t))
    assert tuple(t) == (1, 0, 0)
    destroy(c, plan)


@pytest.mark.parametrize("inplace", [False, True])
def test_r2c_must_transform_z(inplace):
    for P, decomp, p1, p2 in ((1, SL, 1, 1), (4, PE, 2, 2)):
        c, plan = create(0, P, decomp, R2C, (8, 16, 32), p1, p2, inplace=inplace)
        for m in MASKS:
            assert set_axes(plan, m) == (0 if m[2] else ERR_INVALID), m
        destroy(c, plan)


def test_r2r_kinds_still_reported():
    c, plan = create(0, 1, SL, None, (8, 16, 32), 1, 1, kinds=MIXED)
    assert set_axes(plan, (0, 1, 1)) == 0
    k = (C.c_int * 3)()
    check(lib().dfft_plan_get_r2r_kinds(plan, k))
    assert tuple(k) == MIXED
    sc = json.loads(describe_raw(plan, 0, 3))
    assert sc["transform_axes"] == [0, 1, 1]
    destroy(c, plan)


PLANS = [  # transform, kinds
    (C2C, None), (R2C, None), (DCT, None), (None, MIXED),
]


@pytest.mark.parametrize("transform,kinds", PLANS, ids=["c2c", "r2c", "dct", "mixed"])
@pytest.mark.parametrize("P,decomp,p1,p2", [(1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2)])
def test_all_transformed_descriptions_are_unchanged(P, decomp, p1, p2, transform, kinds):
    for comm, send in ((P2P, SYNC), (A2A, SYNC), (P2P, STREAMS)):
        for batch, inplace in ((1, False), (3, False), (1, True)):
            for rank in sorted({0, P - 1}):
                a = create(rank, P, decomp, transform, (16, 32, 64), p1, p2, comm, send, batch, inplace, kinds=kinds)
                b = create(rank, P, decomp, transform, (16, 32, 64), p1, p2, comm, send, batch, inplace, kinds=kinds)
                assert set_axes(b[1], (1, 1, 1)) == 0
                for inverse in (0, 1):
                    for d in (1, 2, 3):
                        da, db = describe_raw(a[1], inverse, d), describe_raw(b[1], inverse, d)
                        assert da == db, (comm, send, batch, inplace, rank, inverse, d)
                        assert "transform_axes" not in da and '"kind":6' not in da and '"kind":7' not in da
                destroy(*a)
                destroy(*b)


# ---- references ---------------------------------------------------------------------------------------------------------
def fwd_ref(x, transform, kinds, axes, d):
    """the transformed axes among the first d stages (z, y, x order), forward"""
    for axis in (2, 1, 0)[:d]:
        if not axes[axis]:
            continue
        if kinds is not None:
            x = r2r_1d(x, kinds[axis], False, axis)
        elif transform == R2C and axis == 2:
            x = np.fft.rfft(x, axis=2)
        else:
            x = np.fft.fft(x, axis=axis)
    return x


def inv_ref(X, transform, kinds, axes, d, nz):
    """the unnormalised inverse of fwd_ref (z last: C2R ends real)"""
    for axis in (0, 1, 2):
        if axis not in (2, 1, 0)[:d] or not axes[axis]:
            continue
        if kinds is not None:
            X = r2r_1d(X, kinds[axis], True, axis)
        elif transform == R2C and axis == 2:
            X = np.fft.irfft(X, n=nz, axis=2) * nz
        else:
            X = np.fft.ifft(X, axis=axis) * X.shape[axis]
    return X


class RealMemory(Memory):
    def add(self, base, nelem):
        arr = np.zeros(nelem, dtype=np.float64)
        self.regions.append((base, arr))
        return arr


def pass_result(st, data, kind_default):
    """what pass st stores for its loaded lines data[a0, a1, n, b] (n-point lines along axis 2)"""
    k = st["kind"]
    if k in (6, 7):
        return data.copy()
    if k in (0, 1):
        return np.fft.ifft(data, axis=2) * data.shape[2] if st["inverse"] else np.fft.fft(data, axis=2)
    if k in (4, 5):
        return r2r_1d(data, KIND[st.get("r2r", kind_default)], st["inverse"], 2)
    raise AssertionError(f"unexpected pass kind {k}")


def run(P, decomp, transform, shape, p1, p2, axes, inverse, d, comm=P2P, send=SYNC, kinds=None, batch=1, inplace=False, scale=None,
        prec=dfft.F64, mutate=None):
    """replays every rank's steps in lock step; returns the worst rel-L2 error of any rank's output block"""
    nx, ny, nz = shape
    scheds = [describe(r, P, decomp, transform, shape, p1, p2, axes, inverse, d, comm, send, batch, inplace, scale, prec, kinds) for r in range(P)]
    if mutate:
        mutate(scheds)
    real = kinds is not None
    r2c = transform == R2C
    es = scheds[0]["esize"]
    assert not scheds[0]["overlapped"]
    if axes != (1, 1, 1):
        assert scheds[0]["transform_axes"] == list(axes)
    lay = lambda r, w: dfft.layout(decomp, DCT if real else transform, nx, ny, nz, p1, p2, r, w)
    rng = np.random.default_rng(P * 1000 + nx + ny + nz + batch + 17 * axes[0] + 5 * axes[1] + axes[2] + 3 * d)
    if real or r2c:
        xg = rng.standard_normal((batch,) + shape)
    else:
        xg = rng.standard_normal((batch,) + shape) + 1j * rng.standard_normal((batch,) + shape)
    spec = np.stack([fwd_ref(xg[f], transform, kinds, axes, d) for f in range(batch)])
    src_g = spec if inverse else xg
    want_g = np.stack([inv_ref(spec[f], transform, kinds, axes, d, nz) for f in range(batch)]) if inverse else spec
    s_used = 1.0 if scale is None else scale[1 if inverse else 0]
    if prec == dfft.F32:
        s_used = float(np.float32(s_used))
    mem = RealMemory(es) if real else Memory(es)
    for r in range(P):
        for s_ in range(scheds[r]["nslots"]):
            mem.add(scheds[r]["slots"][s_][r], scheds[r]["slot_bytes"] // es)
    src_w, dst_w = (d, 0) if inverse else (0, d)
    # R2C: the real side is stored as complex pairs, like the kernels read it
    real_side_in, real_side_out = r2c and not inverse, r2c and bool(inverse)
    uout = []
    for r in range(P):
        isz, ist = lay(r, src_w)
        osz, ost = lay(r, dst_w)
        ni = int(np.prod(isz)) // (2 if real_side_in else 1)
        no = int(np.prod(osz)) // (2 if real_side_out else 1)
        if batch > 1:
            fi, fo = scheds[r]["field_in"] // es, scheds[r]["field_out"] // es
        else:
            fi, fo = (scheds[r]["domain_bytes"] // es,) * 2 if inplace else (ni, no)
        a = mem.add(USER_IN + (r << 48), max(batch * max(fi, ni), 1))
        for f in range(batch):
            blk = np.ascontiguousarray(src_g[f][ist[0]:ist[0] + isz[0], ist[1]:ist[1] + isz[1], ist[2]:ist[2] + isz[2]]).ravel()
            a[f * fi:f * fi + ni] = blk.view(np.complex128) if real_side_in else blk
        uout.append((a, fo, no) if inplace else (mem.add(USER_OUT + (r << 48), max(batch * max(fo, no), 1)), fo, no))
    nsteps = len(scheds[0]["steps"])
    assert all(len(s["steps"]) == nsteps for s in scheds)
    order = Ordering(scheds)
    scaled = {}  # output array -> how often each element was scaled
    for k in range(nsteps):
        pending = []
        for r in range(P):
            st = scheds[r]["steps"][k]
            if st["type"] == 1:
                continue
            if st["type"] == 2:
                sb = scheds[r]["slots"][st["send_slot"]][r]
                for peer in st["peers"]:
                    q = peer["rank"]
                    rb = scheds[q]["slots"][st["recv_slot"]][q]
                    mine = [pp for pp in scheds[q]["steps"][k]["peers"] if pp["rank"] == r][0]
                    assert mine["rcount"] == peer["scount"]
                    src, so = mem.resolve(sb + peer["soff"] * es)
                    dst, do = mem.resolve(rb + mine["roff"] * es)
                    order.read(r, k, id(src), src.size, np.arange(so, so + peer["scount"]))
                    pending.append((dst, np.arange(do, do + peer["scount"]), src[so:so + peer["scount"]].copy(), q))
                continue
            kind = st["kind"]
            if kind in (6, 7):
                assert "n" in st and st["log2n"] == 0 and "r2r" not in st
                assert st["label"].split()[0] in "xyz" and "copy" in st["label"]
            N = st.get("n", 1 << st["log2n"])
            A0, A1, B = st["A0"], st["A1"], st["B"]
            ub_in = {1: USER_IN, 2: USER_IN if inplace else USER_OUT}.get(st["in_user"])
            ub_in = None if ub_in is None else ub_in + (r << 48)
            ub_out = (USER_IN if inplace else USER_OUT) + (r << 48) if st["out_user"] == 2 else None
            n_in, n_out = (N + 1, N) if kind == 3 else (N, N + 1) if kind == 2 else (N, N)
            data = np.zeros((A0, A1, n_in, B), dtype=np.float64 if real else np.complex128)
            for base, ns, off in view_indices(st["in"], A0, A1, n_in, B, ub_in):
                arr, o = mem.resolve(base)
                data[:, :, ns, :] = arr[o + off]
                order.read(r, k, id(arr), arr.size, o + off)
            if kind == 2:  # R2C: N complex = 2N reals in, N+1 complex out
                res = np.fft.rfft(np.ascontiguousarray(data[..., 0]).view(np.float64), axis=2)[..., None]
            elif kind == 3:
                res = np.ascontiguousarray(np.fft.irfft(data[..., 0], n=2 * N, axis=2) * (2 * N)).view(np.complex128)[..., None]
            else:
                res = pass_result(st, data, scheds[r].get("r2r"))
            if "scale" in st:
                res = res * st["scale"]
            for base, ns, off in view_indices(st["out"], A0, A1, n_out, B, ub_out):
                arr, o = mem.resolve(base)
                pending.append((arr, o + off, res[:, :, ns, :], r))
                if "scale" in st:
                    assert ub_out is not None, "only stores into the caller's output are scaled"
                    scaled.setdefault(id(arr), np.zeros(arr.size, dtype=np.int64))
                    np.add.at(scaled[id(arr)], (o + off).ravel(), 1)
        for arr, idx, val, who in pending:
            order.write(who, k, id(arr), arr.size, idx)
            arr[idx] = val
    worst = 0.0
    for r in range(P):
        osz, ost = lay(r, dst_w)
        arr, fo, no = uout[r]
        for f in range(batch):
            got = arr[f * fo:f * fo + no]
            got = (got.view(np.float64) if real_side_out else got).reshape(osz)
            want = want_g[f][ost[0]:ost[0] + osz[0], ost[1]:ost[1] + osz[1], ost[2]:ost[2] + osz[2]] * s_used
            worst = max(worst, float(np.linalg.norm(got - want) / np.linalg.norm(want)))
            if scale is not None and s_used != 1.0:
                cnt = scaled.get(id(arr), np.zeros(arr.size, dtype=np.int64))[f * fo:f * fo + no]
                assert (cnt == 1).all(), f"rank {r} field {f}: an output value is scaled {int(cnt.min())}..{int(cnt.max())} times"
    return worst


# ---- replays --------------------------------------------------------------------------------------------------------------
GRIDS = [  # P, decomp, shape, p1, p2, comm
    (1, SL, (8, 16, 64), 1, 1, P2P),    # one rank, blocked hand-over
    (1, ZY, (8, 16, 32), 1, 1, P2P),
    (1, PE, (8, 16, 32), 1, 1, A2A),
    (3, SL, (8, 16, 64), 3, 1, A2A),    # uneven splits
    (4, ZY, (8, 4, 32), 4, 1, P2P),
    (5, SL, (16, 16, 128), 5, 1, P2P),  # uneven, blocked with a tail
    (6, PE, (8, 16, 32), 2, 3, A2A),    # z split into odd column counts
    (8, PE, (8, 16, 32), 2, 4, P2P),
    (4, PE, (8, 16, 32), 4, 1, P2P),    # P2 = 1: the z pass stays on its rank (rule 3 drops a kept z)
    (3, PE, (8, 16, 32), 3, 1, A2A),    # 8 over 3
    (4, PE, (8, 16, 32), 1, 4, A2A),    # P1 = 1
]


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_c2c_every_mask(axes, inverse):
    for P, decomp, shape, p1, p2, comm in GRIDS:
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, comm) < 1e-12, (P, decomp)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_mixed_r2r_every_mask(axes, inverse):
    for P, decomp, shape, p1, p2, comm in GRIDS:
        assert run(P, decomp, None, shape, p1, p2, axes, inverse, 3, comm, kinds=MIXED) < 1e-12, (P, decomp)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", R2C_MASKS, ids=mask_id)
def test_replay_r2c_masks(axes, inverse):
    for P, decomp, shape, p1, p2, comm in GRIDS + [(4, SL, (8, 16, 128), 4, 1, P2P), (8, PE, (16, 16, 2048), 4, 2, P2P)]:
        assert run(P, decomp, R2C, shape, p1, p2, axes, inverse, 3, comm) < 1e-12, (P, decomp)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", [(0, 1, 1), (1, 1, 0), (0, 0, 0), (1, 0, 1)], ids=mask_id)
@pytest.mark.parametrize("P,decomp,shape,p1,p2,comm,send", R2R_CASES)
def test_replay_every_rank_count(P, decomp, shape, p1, p2, comm, send, axes, inverse):
    """1-8 ranks, every decomposition, P2P and A2A, Streams plans (sequential), odd column counts, blocked tails"""
    assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, comm, send) < 1e-12
    assert run(P, decomp, None, shape, p1, p2, axes, inverse, 3, comm, send, kinds=MIXED) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_partial(axes, inverse, d):
    """partial d: the first d stages in z, y, x order, each transformed or kept"""
    for P, decomp, shape, p1, p2, comm in ((1, SL, (8, 16, 64), 1, 1, P2P), (3, SL, (8, 16, 64), 3, 1, A2A), (6, PE, (8, 16, 32), 2, 3, P2P),
                                           (1, PE, (8, 16, 32), 1, 1, A2A)):
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, d, comm) < 1e-12
        assert run(P, decomp, None, shape, p1, p2, axes, inverse, d, comm, kinds=MIXED) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_bluestein(axes, inverse):
    for P, decomp, shape, p1, p2, comm in ((1, SL, (12, 10, 7), 1, 1, P2P), (1, SL, (6, 100, 130), 1, 1, P2P), (2, SL, (6, 100, 130), 2, 1, P2P),
                                           (1, ZY, (6, 12, 7), 1, 1, P2P), (3, ZY, (12, 10, 7), 3, 1, A2A), (6, PE, (12, 10, 7), 2, 3, P2P)):
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, comm) < 1e-12


S = (0.25, 1.0 / 3.0)


@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("axes", MASKS, ids=mask_id)
def test_replay_batch_inplace_scale(axes, inverse):
    """batch 3, in-place plans and a scale that is not 1: every output value scaled exactly once"""
    for P, decomp, shape, p1, p2 in ((1, SL, (8, 16, 64), 1, 1), (1, ZY, (8, 16, 32), 1, 1), (1, PE, (8, 16, 32), 1, 1),
                                     (3, SL, (8, 16, 64), 3, 1), (4, PE, (8, 16, 32), 2, 2), (3, ZY, (8, 4, 16), 3, 1)):
        for d in (1, 3) if decomp == ZY else (1, 2, 3):  # Z_Then_YX: partial inverses are not offered
            assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, d, batch=3, scale=S) < 1e-12
            assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, d, inplace=True, scale=S) < 1e-12
            assert run(P, decomp, None, shape, p1, p2, axes, inverse, d, kinds=MIXED, inplace=True, batch=3, scale=S) < 1e-12
        assert run(P, decomp, C2C, shape, p1, p2, axes, inverse, 3, scale=S, prec=dfft.F32) < 1e-12
        if axes[2]:
            assert run(P, decomp, R2C, shape, p1, p2, axes, inverse, 3, batch=3, scale=S) < 1e-12


# ---- elision ------------------------------------------------------------------------------------------------------------
def same_view(st, inplace):
    """the same elements of the same buffer (in place, the caller's `in` and `out` are one buffer)"""
    return st["in"] == st["out"] and (st["in_user"] == st["out_user"] or (inplace and st["in_user"] > 0 and st["out_user"] > 0))


ELIDE_GRIDS = [(1, SL, 1, 1), (1, ZY, 1, 1), (1, PE, 1, 1), (4, SL, 4, 1), (4, ZY, 4, 1), (4, PE, 2, 2), (3, SL, 3, 1), (4, PE, 4, 1),
               (4, PE, 1, 4)]


@pytest.mark.parametrize("inplace", [False, True])
@pytest.mark.parametrize("transform,kinds", [(C2C, None), (None, MIXED)], ids=["c2c", "mixed"])
def test_elision_rules(transform, kinds, inplace):
    shape = (8, 16, 64)
    for P, decomp, p1, p2 in ELIDE_GRIDS:
        for axes in MASKS:
            for inverse in (0, 1):
                for d in (1, 2, 3):
                    sc = describe(0, P, decomp, transform, shape, p1, p2, axes, inverse, d, inplace=inplace, kinds=kinds)
                    passes = [s for s in sc["steps"] if s["type"] == 0]
                    for st in passes:
                        if st["kind"] in (6, 7):
                            # rule 1: a copy that moves nothing stays only where it stores final values in place (it applies
                            # the scale)
                            assert not same_view(st, inplace) or (inplace and st["out_user"] == 2), (P, decomp, axes, inverse, d, st["label"])
                    labels = [s["label"] for s in passes]
                    # rule 3: the z pass is local on one rank, on slab ZY_Then_X and on pencil grids with P2 = 1
                    z_local = P == 1 or decomp == SL or (decomp == PE and p2 == 1)
                    if not axes[2] and d >= 2:
                        assert any(l.startswith("z ") for l in labels) != z_local, (P, decomp, p1, p2, axes, inverse, d, labels)
                    if P == 1 and not axes[0] and d == 3:  # rule 2
                        d2 = describe(0, P, decomp, transform, shape, p1, p2, axes, inverse, 2, inplace=inplace, kinds=kinds)
                        assert sc["steps"] == d2["steps"], (decomp, axes, inverse)
                        assert not any(l.startswith("x ") for l in labels)
                    if P == 1 and axes == (1, 1, 0) and d == 3:
                        assert sorted(labels) == ["x pass", "y pass"]


def test_one_rank_masks_need_few_passes():
    """one rank: each kept axis saves its pass except a kept y between two transformed axes"""
    for decomp in (SL, ZY, PE):
        for axes in MASKS:
            for inverse in (0, 1):
                sc = describe(0, 1, decomp, C2C, (8, 16, 64), 1, 1, axes, inverse, 3)
                passes = [s for s in sc["steps"] if s["type"] == 0]
                assert len(passes) <= 3 - (not axes[0]) - (not axes[2]) + (axes == (0, 0, 0)), (decomp, axes, inverse, [s["label"] for s in passes])
                assert sum(s["kind"] in (6, 7) for s in passes) <= 1


def test_streams_plans_run_sequential_schedule():
    for axes in ((0, 1, 1), (1, 0, 1), (1, 1, 0)):
        for inverse in (0, 1):
            sc = describe(0, 4, SL, C2C, (16, 8, 64), 4, 1, axes, inverse, 3, send=STREAMS)
            assert not sc["overlapped"] and all(s["stream"] == 0 for s in sc["steps"])
            sc = describe(0, 4, PE, C2C, (16, 8, 64), 2, 2, axes, inverse, 3, send=STREAMS)
            assert not sc["overlapped"]


def test_fused_and_batched_stages_need_every_axis():
    """the fused z + y stage (512^3 one-rank slab) and the batched stage (32^3) are not chosen with a kept axis"""
    for axes in ((0, 1, 1), (1, 1, 0), (1, 0, 1)):
        for inverse in (0, 1):
            sc = describe(0, 1, SL, C2C, (512, 512, 512), 1, 1, axes, inverse, 3)
            assert all(s["label"] not in ("zy pass: z phase", "yz pass: z phase") for s in sc["steps"])
            sc = describe(0, 1, SL, C2C, (32, 32, 32), 1, 1, axes, inverse, 3, batch=4)
            assert all(not s["label"].startswith("batched") for s in sc["steps"])
    full = describe(0, 1, SL, C2C, (512, 512, 512), 1, 1, None, 0, 3)
    assert any(s["label"] == "zy pass: z phase" for s in full["steps"])


def _break_copy(scheds):
    for sc in scheds:
        for st in sc["steps"]:
            if st["type"] == 0 and st["kind"] in (6, 7):
                st["out"]["segs"][0]["sA0"], st["out"]["sN"] = st["out"]["sN"], st["out"]["segs"][0]["sA0"]
                return


def test_replay_rejects_a_broken_copy():
    """negative test: a copy step with its output strides swapped does not reproduce the reference"""
    assert run(1, PE, C2C, (8, 16, 32), 1, 1, (1, 0, 1), 0, 3) < 1e-12
    try:
        err = run(1, PE, C2C, (8, 16, 32), 1, 1, (1, 0, 1), 0, 3, mutate=_break_copy)
    except (AssertionError, KeyError, IndexError):
        return
    assert err > 1e-3
