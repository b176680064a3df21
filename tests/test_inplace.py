"""In-place plans (dfft_plan_create_inplace) without a GPU: argument checks, the work area, and CPU replays of every rank's
step list with the caller's `in` and `out` mapped to ONE address range.

The replay is the numpy machinery of test_schedule_emulation.py with three additions:
  - the buffer of a rank holds `batch` fields dfft_get_domain_size() bytes apart; real rows of R2C / C2R plans are padded
    to Nz/2 + 1 complex units, and the padding must never be read or written;
  - the happens-before check (Ordering) now also sees the read-after-write and write-after-read pairs on the buffer;
  - a line check inside every step: a line may only write addresses that it reads itself or that no other line of the
    step reads (the passes load a line or tile completely before they store it, so that is what in place needs), and the
    two phases of the fused z + y stage and of the one-launch batched stage, which run concurrently, touch disjoint
    planes / fields."""
import ctypes as C
import json

import numpy as np
import pytest

import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from oracle import dft_oracle as O

from test_schedule_emulation import A2A, P2P, PE, SL, STREAMS, SYNC, ZY, Memory, Ordering, view_indices

USER = 1 << 60  # synthetic address range of the caller's one buffer (rank r: USER + r << 48)
SIZE_MAX = (1 << 64) - 1
PAD = 1234.5 - 678.25j  # value of the padding of real rows


def create(rank, P, decomp, transform, shape, p1, p2, batch=1, comm=P2P, send=SYNC, prec=None, inplace=True):
    """dry plan: (rc, message, comm, plan)"""
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(rank, P, C.byref(c)))
    cfg = _lib.dfft_config(1, 0, comm, send, None, comm, send)
    plan = C.c_void_p()
    fn = lib().dfft_plan_create_inplace if inplace else lib().dfft_plan_create_batched
    rc = fn(c, C.byref(cfg), decomp, dfft.F64 if prec is None else prec, transform, *shape, p1, p2, batch, 1, C.byref(plan))
    return rc, (lib().dfft_last_error_string() or b"").decode(), c, plan


def describe(rank, P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, prec=None, scale=None, inplace=True):
    rc, msg, c, plan = create(rank, P, decomp, transform, shape, p1, p2, batch, comm, send, prec, inplace)
    assert rc == 0, msg
    if scale is not None:
        assert lib().dfft_plan_set_scale(plan, *scale) == 0
    need = C.c_size_t()
    check(lib().dfft_plan_describe(plan, inverse, d, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib().dfft_plan_describe(plan, inverse, d, buf, need.value, C.byref(need)))
    sc = json.loads(buf.value.decode())
    sc["domain_bytes"] = lib().dfft_get_domain_size(plan)
    sc["work_bytes"] = lib().dfft_get_work_size_device(plan)
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return sc


def _line_check(r, k, st, reads, writes):
    """reads / writes: [(array, flat indices, line ids)] of one step: a line writes only what it reads itself or what no
    other line of the step reads"""
    owner = {}
    for arr, idx, line in reads:
        i, l = np.asarray(idx).ravel(), np.broadcast_to(line, np.shape(idx)).ravel()
        prev = owner.get(id(arr))
        if prev is not None:
            i, l = np.concatenate([prev[0], i]), np.concatenate([prev[1], l])
        owner[id(arr)] = (i, l)
    table = {}
    for key, (i, l) in owner.items():
        u, inv = np.unique(i, return_inverse=True)
        lo = np.full(u.size, np.iinfo(np.int64).max)
        hi = np.full(u.size, -1)
        np.minimum.at(lo, inv, l)
        np.maximum.at(hi, inv, l)
        table[key] = (u, np.where(lo == hi, lo, -2))  # the one reading line, or -2: several lines read it
    for arr, idx, line in writes:
        if id(arr) not in table:
            continue
        u, rl = table[id(arr)]
        i, l = np.asarray(idx).ravel(), np.broadcast_to(line, np.shape(idx)).ravel()
        pos = np.searchsorted(u, i)
        hit = (pos < u.size) & (u[np.minimum(pos, u.size - 1)] == i)
        reader = np.where(hit, rl[np.minimum(pos, u.size - 1)], -1)
        bad = (reader != -1) & (reader != l)
        assert not bad.any(), (f"rank {r} step {k} ({st['label']}): line {int(l[bad][0])} writes an element that line {int(reader[bad][0])} "
                               f"reads (or that several lines read)")


def _phase_check(r, k, acc, groups):
    """the two phases of a two-phase kernel (steps k-1 and k): every element is touched by one plane / field only"""
    owner = {}
    for arr, idx, grp in acc:
        i, g = np.asarray(idx).ravel(), np.broadcast_to(grp, np.shape(idx)).ravel()
        prev = owner.get(id(arr))
        owner[id(arr)] = (i, g) if prev is None else (np.concatenate([prev[0], i]), np.concatenate([prev[1], g]))
    for i, g in owner.values():
        u, inv = np.unique(i, return_inverse=True)
        lo = np.full(u.size, groups)
        hi = np.full(u.size, -1)
        np.minimum.at(lo, inv, g)
        np.maximum.at(hi, inv, g)
        assert (lo == hi).all(), f"rank {r} steps {k - 1}/{k}: the two phases of one launch share elements across planes / fields"


def run_inplace(P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch=1, scale=1.0, prec=None, mutate=None):
    """Replays an in-place exec on every rank; returns the worst rel-L2 error of the output against scale times the
    oracle."""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    sc_ = None if scale == 1.0 else ((1.0, scale) if inverse else (scale, 1.0))
    scheds = [describe(r, P, decomp, transform, shape, p1, p2, comm, send, inverse, d, batch, prec, sc_) for r in range(P)]
    if mutate:
        mutate(scheds)  # negative tests
    es = scheds[0]["esize"]
    nzc = nz if c2c else nz // 2 + 1
    lay = lambda r, w: dfft.layout(decomp, transform, nx, ny, nz, p1, p2, r, w)
    xs = [O.complex_input(shape, seed=77 + f) if c2c else O.real_input(shape, seed=77 + f) for f in range(batch)]
    specs = [O.fft_c2c(x, d) if c2c else O.fft_r2c(x, d) for x in xs]
    mem = Memory(es)
    for r in range(P):
        assert scheds[r]["inplace"] is True
        for s_ in range(scheds[r]["nslots"]):
            mem.add(scheds[r]["slots"][s_][r], scheds[r]["slot_bytes"] // es)
    bufs, dom, pads = [], [], []
    for r in range(P):
        D = scheds[r]["domain_bytes"] // es
        if batch > 1:
            assert scheds[r]["field_in"] == scheds[r]["field_out"] == D * es
        dom.append(D)
        buf = mem.add(USER + (r << 48), batch * D)
        isz, ist = lay(r, 0)
        osz, ost = lay(r, d)
        pad = np.zeros(batch * D, dtype=bool)  # padding of the real rows: never read or written
        for f in range(batch):
            if not inverse:
                blk = np.ascontiguousarray(O.block(xs[f], ist, isz))
                if c2c:
                    buf[f * D:f * D + blk.size] = blk.astype(np.complex128).ravel()
                else:  # rows of Nz reals = Nz/2 units, Nzc units apart
                    rows = buf[f * D:f * D + isz[0] * isz[1] * nzc].reshape(isz[0] * isz[1], nzc)
                    rows[:, :nz // 2] = blk.reshape(-1, nz).view(np.complex128)
                    rows[:, nz // 2:] = PAD
            else:
                src = np.ascontiguousarray(O.block(specs[f], ost, osz)).ravel()
                buf[f * D:f * D + src.size] = src
            if not c2c:  # the real input rows (forward) / output rows (inverse)
                m = pad[f * D:f * D + isz[0] * isz[1] * nzc].reshape(-1, nzc)
                m[:, nz // 2:] = True
        bufs.append(buf)
        pads.append(pad)
    nsteps = len(scheds[0]["steps"])
    assert all(len(sc["steps"]) == nsteps for sc in scheds)
    order = Ordering(scheds)
    prev_acc = {}
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
                    src, so = mem.resolve(sb + peer["soff"] * es)
                    dst, do = mem.resolve(rb + mine["roff"] * es)
                    order.read(r, k, id(src), src.size, np.arange(so, so + peer["scount"]))
                    pending.append((dst, do, src[so:so + peer["scount"]].copy(), q))
                continue
            kind = st["kind"]
            N = st.get("n", 1 << st["log2n"])
            A0, A1, B = st["A0"], st["A1"], st["B"]
            ub_in = USER + (r << 48) if st["in_user"] in (1, 2) else None  # `in` and `out` are the same buffer
            ub_out = USER + (r << 48) if st["out_user"] == 2 else None
            n_in, n_out = {0: (N, N), 1: (N, N), 2: (N, N + 1), 3: (N + 1, N)}[kind]
            b_ = B if kind in (0, 1) else 1
            line = (np.arange(A0)[:, None, None, None] * A1 + np.arange(A1)[None, :, None, None]) * b_ + np.arange(b_)[None, None, None, :]
            field = st.get("field", -1)
            reads, writes = [], []
            data = np.zeros((A0, A1, n_in, b_), dtype=np.complex128)
            for base, ns, off in view_indices(st["in"], A0, A1, n_in, b_, ub_in):
                arr, o = mem.resolve(base)
                data[:, :, ns, :] = arr[o + off]
                order.read(r, k, id(arr), arr.size, o + off)
                reads.append((arr, o + off, line))
            for base, ns, off in view_indices(st["out"], A0, A1, n_out, b_, ub_out):
                arr, o = mem.resolve(base)
                writes.append((arr, o + off, line, ns))
            _line_check(r, k, st, reads, [w[:3] for w in writes])
            for j, (arr, idx, _) in enumerate(reads + [w[:3] for w in writes]):
                if arr is not bufs[r] or idx.size == 0:  # empty tail passes of ranks without leftover columns
                    continue
                if field >= 0:  # a per-field step stays inside its field
                    assert field * dom[r] <= idx.min() and idx.max() < (field + 1) * dom[r], f"step {k} leaves field {field}"
                # forward: the padding of the real input rows is not read (until a complex pass has stored there);
                # inverse: the C2R pass does not store into it
                is_read = j < len(reads)
                if (is_read and not inverse) or (not is_read and kind == 3):
                    assert not pads[r][idx].any(), f"rank {r} step {k} ({st['label']}) touches the padding of a real row"
                elif not inverse:
                    pads[r][idx] = False
            # the fused z + y stage and the batched stage: both listed phases run concurrently (planes / fields apart)
            two_phase = st["label"].startswith(("zy pass", "yz pass", "batched pass"))
            if two_phase:
                groups = batch if st["label"].startswith("batched") else nx
                grp = np.arange(A0)[:, None, None, None] * groups // A0
                acc = [(a, i, grp) for a, i, _ in reads + [w[:3] for w in writes]]
                if prev_acc.get(r) is not None:
                    _phase_check(r, k, prev_acc[r] + acc, groups)
                    prev_acc[r] = None if not st["label"].startswith("batched") else acc
                else:
                    prev_acc[r] = acc
            else:
                prev_acc[r] = None
            if kind in (0, 1):
                res = np.fft.ifft(data, axis=2) * N if st["inverse"] else np.fft.fft(data, axis=2)
            elif kind == 2:
                res = np.fft.rfft(np.ascontiguousarray(data[..., 0]).view(np.float64), axis=2)[..., None]
            else:
                reals = np.fft.irfft(data[..., 0], n=2 * N, axis=2) * (2 * N)
                res = np.ascontiguousarray(reals).view(np.complex128)[..., None]
            res = res * st.get("scale", 1.0)
            for arr, idx, _, ns in writes:
                pending.append((arr, idx, res[:, :, ns, :], r))
        for arr, idx, val, who in pending:
            if isinstance(idx, (int, np.integer)):
                order.write(who, k, id(arr), arr.size, np.arange(idx, idx + val.size))
                arr[idx:idx + val.size] = val
            else:
                order.write(who, k, id(arr), arr.size, idx)
                arr[idx] = val
    worst = 0.0
    for r in range(P):
        D = dom[r]
        if not inverse:
            assert (bufs[r][pads[r]] == PAD).all()
        for f in range(batch):
            if not inverse:
                osz, ost = lay(r, d)
                got = bufs[r][f * D:f * D + int(np.prod(osz))].reshape(osz)
                worst = max(worst, O.rel_l2(got, scale * O.block(specs[f], ost, osz)))
            else:
                isz, ist = lay(r, 0)
                n = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
                want = O.block(xs[f], ist, isz).astype(np.complex128 if c2c else np.float64)
                if c2c:
                    got = bufs[r][f * D:f * D + int(np.prod(isz))].reshape(isz)
                else:
                    rows = bufs[r][f * D:f * D + isz[0] * isz[1] * nzc].reshape(-1, nzc)[:, :nz // 2]
                    got = np.ascontiguousarray(rows).view(np.float64).reshape(isz)
                worst = max(worst, O.rel_l2(got, scale * n * want))
    return worst


# ---- argument checks ------------------------------------------------------------------------------------------------
def _plan_info(P, decomp, transform, shape, p1, p2, inplace, batch=1, comm=P2P):
    rc, msg, c, plan = create(0, P, decomp, transform, shape, p1, p2, batch, comm, SYNC, None, inplace)
    assert rc == 0, msg
    info = dict(inplace=lib().dfft_plan_is_inplace(plan), work=lib().dfft_get_work_size_device(plan), dom=lib().dfft_get_domain_size(plan))
    in_size = (C.c_size_t * 3)()
    out_size = (C.c_size_t * 3)()
    check(lib().dfft_get_in_size(plan, in_size))
    check(lib().dfft_get_out_size(plan, out_size))
    info["in_size"], info["out_size"] = list(in_size), list(out_size)
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    return info


def test_is_inplace():
    assert _plan_info(1, SL, dfft.C2C, (8, 8, 8), 1, 1, True)["inplace"] == 1
    assert _plan_info(1, SL, dfft.C2C, (8, 8, 8), 1, 1, False)["inplace"] == 0
    assert lib().dfft_plan_is_inplace(None) == 0


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm", [
    (1, SL, dfft.C2C, (64, 32, 16), 1, 1, P2P), (1, ZY, dfft.R2C, (16, 8, 32), 1, 1, P2P), (1, PE, dfft.C2C, (8, 16, 32), 1, 1, P2P),
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P), (4, SL, dfft.R2C, (16, 8, 64), 4, 1, A2A), (6, PE, dfft.R2C, (8, 16, 16), 3, 2, A2A),
    (4, ZY, dfft.C2C, (8, 4, 16), 4, 1, P2P)])
def test_work_area(P, decomp, transform, shape, p1, p2, comm):
    """one rank: one slot, half the out-of-place work area; several ranks: the out-of-place slots"""
    ip = describe(0, P, decomp, transform, shape, p1, p2, comm, SYNC, 0, 3)
    oop = describe(0, P, decomp, transform, shape, p1, p2, comm, SYNC, 0, 3, inplace=False)
    assert ip["inplace"] is True and "inplace" not in oop
    assert ip["slot_bytes"] == oop["slot_bytes"] and ip["domain_bytes"] == oop["domain_bytes"]
    if P == 1:
        assert ip["nslots"] == 1 and oop["nslots"] == 2
        assert ip["work_bytes"] == ip["slot_bytes"] == oop["work_bytes"] // 2
    else:
        assert ip["nslots"] == oop["nslots"] >= 2 and ip["work_bytes"] == oop["work_bytes"]


@pytest.mark.parametrize("P,decomp,shape,p1,p2", [(1, SL, (8, 16, 64), 1, 1), (3, SL, (8, 16, 16), 3, 1), (4, ZY, (8, 4, 32), 4, 1),
                                                  (6, PE, (8, 16, 16), 3, 2), (8, PE, (16, 16, 2048), 4, 2), (2, PE, (4, 4, 4), 1, 2)])
def test_domain_covers_the_padded_input(P, decomp, shape, p1, p2):
    """dfft_get_domain_size covers the padded real input ([X][Y][Nz/2+1] complex units) and every other layout of every
    rank; the getters keep the logical sizes"""
    nzc = shape[2] // 2 + 1
    for r in range(P):
        rc, msg, c, plan = create(r, P, decomp, dfft.R2C, shape, p1, p2)
        assert rc == 0, msg
        dom = lib().dfft_get_domain_size(plan)
        in_size = (C.c_size_t * 3)()
        check(lib().dfft_get_in_size(plan, in_size))
        assert in_size[2] == shape[2]
        assert dom >= in_size[0] * in_size[1] * nzc * 16
        for w in (1, 2, 3):
            assert dom >= int(np.prod(dfft.layout(decomp, dfft.R2C, *shape, p1, p2, r, w)[0])) * 16
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)


def test_batch_validation():
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, batch=0)
    assert rc == -1 and "batch" in msg
    lib().dfft_comm_destroy(c)
    # a field is domain_size = 8^3 * 16 bytes: one field too many overflows size_t
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, batch=SIZE_MAX // (8 ** 3 * 16) + 1)
    assert rc == -1 and "overflows" in msg
    lib().dfft_comm_destroy(c)
    rc, msg, c, plan = create(0, 1, SL, dfft.C2C, (8, 8, 8), 1, 1, batch=SIZE_MAX // (8 ** 3 * 16))
    assert rc == 0, msg
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(c)
    # R2C: the padded input of an in-place plan is larger than the logical one
    rc, msg, c, plan = create(0, 1, SL, dfft.R2C, (8, 8, 8), 1, 1, batch=SIZE_MAX // (8 * 8 * 5 * 16) + 1)
    assert rc == -1 and "overflows" in msg
    lib().dfft_comm_destroy(c)


def test_step_lists_mark_the_buffer():
    """one rank, forward: the z pass runs in place in the buffer, the y pass reads it into the slot, the x pass writes it
    back; inverse: x pass buffer -> slot, y pass slot -> buffer, z pass in place"""
    fwd = describe(0, 1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3)["steps"]
    assert [(s["label"], s["in_user"], s["out_user"]) for s in fwd] == [("z pass", 1, 2), ("y pass", 2, 0), ("x pass", 0, 2)]
    inv = describe(0, 1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 1, 3)["steps"]
    assert [(s["label"], s["in_user"], s["out_user"]) for s in inv] == [("x pass", 1, 0), ("y pass", 0, 2), ("z pass", 2, 2)]
    # padded real rows: R2C input lines and C2R output lines are Nz/2 + 1 complex units apart
    r2c = describe(0, 1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC, 0, 3)["steps"][0]
    assert r2c["kind"] == 2 and r2c["in"]["segs"][0]["sA1"] == 129 and r2c["out"]["segs"][0]["sA1"] == 129
    c2r = describe(0, 1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC, 1, 3)["steps"][-1]
    assert c2r["kind"] == 3 and c2r["in"]["segs"][0]["sA1"] == 129 and c2r["out"]["segs"][0]["sA1"] == 129
    # the scale is on the steps that store the final values only
    sc = describe(0, 1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3, scale=(0.5, 1.0))["steps"]
    assert ["scale" in s for s in sc] == [False, False, True]


# ---- replays --------------------------------------------------------------------------------------------------------
CASES = [
    # P, decomp, transform, shape, p1, p2, comm, send
    (1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC),          # blocked hand-over, one slot
    (1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC),          # padded rows, blocked + tail column
    (1, ZY, dfft.C2C, (8, 8, 16), 1, 1, P2P, SYNC),
    (1, ZY, dfft.R2C, (8, 4, 32), 1, 1, P2P, SYNC),
    (1, PE, dfft.C2C, (8, 8, 16), 1, 1, P2P, SYNC),
    (1, PE, dfft.R2C, (8, 16, 64), 1, 1, P2P, SYNC),
    (2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS),       # overlapped slab
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, P2P, SYNC),
    (3, SL, dfft.R2C, (8, 16, 16), 3, 1, P2P, SYNC),          # uneven split
    (3, SL, dfft.R2C, (16, 16, 64), 3, 1, P2P, STREAMS),      # uneven, overlapped, tail column
    (8, SL, dfft.C2C, (16, 16, 64), 8, 1, A2A, SYNC),
    (8, SL, dfft.R2C, (16, 8, 64), 8, 1, P2P, STREAMS),       # overlapped + blocked + tail
    (4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, SYNC),         # blocked + tail column (Nzc = 65)
    (4, ZY, dfft.R2C, (8, 4, 32), 4, 1, P2P, SYNC),
    (3, ZY, dfft.C2C, (8, 4, 16), 3, 1, A2A, SYNC),
    (8, PE, dfft.R2C, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 16), 4, 2, A2A, SYNC),
    (6, PE, dfft.R2C, (8, 16, 16), 3, 2, P2P, SYNC),          # uneven
    (8, PE, dfft.R2C, (16, 16, 2048), 4, 2, P2P, SYNC),       # blocked second transposition with tail columns
]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("batch", [1, 3])
def test_inplace_schedules(P, decomp, transform, shape, p1, p2, comm, send, inverse, batch):
    assert run_inplace(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, batch) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_inplace_partial(d, inverse, comm):
    assert run_inplace(8, PE, dfft.R2C, (8, 16, 32), 2, 4, comm, SYNC, inverse, d) < 1e-12
    assert run_inplace(4, PE, dfft.C2C, (8, 8, 16), 2, 2, comm, SYNC, inverse, d, batch=3) < 1e-12
    assert run_inplace(1, PE, dfft.R2C, (8, 8, 16), 1, 1, comm, SYNC, inverse, d) < 1e-12
    assert run_inplace(1, PE, dfft.C2C, (8, 8, 16), 1, 1, comm, SYNC, inverse, d, batch=3, scale=3.0) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_scale(inverse):
    """a scale that is not 1 lands on every output value exactly once, also where the buffer holds intermediates"""
    assert run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, inverse, 3, batch=3, scale=3.0) < 1e-12
    assert run_inplace(1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC, inverse, 3, scale=0.25) < 1e-12
    assert run_inplace(3, SL, dfft.R2C, (16, 16, 64), 3, 1, P2P, STREAMS, inverse, 3, batch=3, scale=3.0) < 1e-12
    assert run_inplace(6, PE, dfft.R2C, (8, 16, 16), 3, 2, A2A, SYNC, inverse, 3, scale=3.0) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_overlapped_pencil(inverse, monkeypatch):
    """overlapped pencil schedules, built without the plan-time measurement that selects the inverse one"""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    assert run_inplace(8, PE, dfft.C2C, (16, 32, 256), 2, 4, P2P, STREAMS, inverse, 3) < 1e-12
    assert run_inplace(4, PE, dfft.R2C, (8, 16, 128), 2, 2, P2P, STREAMS, inverse, 3, batch=3) < 1e-12
    assert run_inplace(8, PE, dfft.R2C, (16, 16, 2048), 4, 2, P2P, STREAMS, inverse, 3) < 1e-12


@pytest.mark.parametrize("shape,batch,prec", [((256, 256, 256), 1, dfft.F64), ((512, 256, 256), 1, dfft.F32), ((32, 32, 32), 3, dfft.F64),
                                              ((64, 64, 64), 2, dfft.F32)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_fused_and_batched_stages(shape, batch, prec, inverse):
    """the fused z + y stage in place (forward: phase A z lines in place, phase B y tiles into the slot; inverse: phase A
    y tiles into the buffer, phase B z lines in place) and the one-launch batched stage with in == out"""
    sc = describe(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec)
    labels = [(s["label"], s["in_user"], s["out_user"]) for s in sc["steps"]]
    if batch > 1:
        assert labels == ([("batched pass: x lines", 1, 2), ("batched pass: y lines", 2, 2), ("batched pass: z lines", 2, 2)] if inverse else
                          [("batched pass: z lines", 1, 2), ("batched pass: y lines", 2, 2), ("batched pass: x lines", 2, 2)])
    elif inverse:
        assert labels == [("x pass", 1, 0), ("yz pass: y phase", 0, 2), ("yz pass: z phase", 2, 2)]
    else:
        assert labels == [("zy pass: z phase", 1, 2), ("zy pass: y phase", 2, 0), ("x pass", 0, 2)]
    if shape[0] <= 64 or shape == (256, 256, 256):
        assert run_inplace(1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, scale=0.5, prec=prec) < 1e-12


@pytest.mark.parametrize("inverse", [0, 1])
def test_inplace_bluestein(inverse):
    """a shape with lengths that are not powers of two (Bluestein passes, sequential schedule)"""
    assert run_inplace(1, SL, dfft.C2C, (12, 10, 7), 1, 1, P2P, SYNC, inverse, 3, batch=2, scale=3.0) < 1e-12
    assert run_inplace(3, PE, dfft.C2C, (12, 10, 7), 3, 1, A2A, SYNC, inverse, 3) < 1e-12


def _shift_rows(label):
    """schedule mutation: the in-place pass `label` stores every line one row further on (into the next line's input)"""
    def mutate(scheds):
        for sc in scheds:
            for st in sc["steps"]:
                if st["type"] == 0 and st["label"] == label:
                    seg = st["out"]["segs"][0]
                    seg["base"] += seg["sA1"] * sc["esize"]
    return mutate


def test_line_check_catches_cross_line_writes():
    """the line check is not vacuous: a z pass that stores each line into the next line's row is rejected (its last line
    would also leave the buffer's field, but the check fires first)"""
    assert run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3) < 1e-12
    with pytest.raises(AssertionError, match="writes an element that line"):
        run_inplace(1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC, 0, 3, mutate=_shift_rows("z pass"))


def test_ordering_check_sees_the_buffer(monkeypatch):
    """the happens-before check covers the shared buffer: an overlapped slab schedule whose exchange stream no longer
    waits for the z pass (whose input the x pass overwrites in place) is rejected"""
    def drop_waits(scheds):
        for sc in scheds:
            for st in sc["steps"]:
                if st["stream"] != 0:
                    st["waits"] = []
    assert run_inplace(2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS, 0, 3) < 1e-12
    with pytest.raises(AssertionError, match="without"):
        run_inplace(2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS, 0, 3, mutate=drop_waits)
