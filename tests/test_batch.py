"""Batched plans (dfft_plan_create_batched) without a GPU: argument checks, the batch = 1 identity, the selection of the
one-launch batched stage, its work list, and CPU replays of batched schedules.

The replay runs the step lists dfft_plan_describe returns for every rank of a batched plan, with the numpy machinery of
test_schedule_emulation.py (memory model, views, happens-before check), on distinct inputs per field.  Every field's
block must match the oracle, and every step may only touch the caller's memory of its own field (the per-field distance
is the product of the buffer's layout, never the domain size)."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from oracle import dft_oracle as O

from test_schedule_emulation import A2A, P2P, PE, SL, STREAMS, SYNC, USER_IN, USER_OUT, ZY, Memory, Ordering, describe, view_indices

HERE = os.path.dirname(os.path.abspath(__file__))
SIZE_MAX = (1 << 64) - 1


def create(rank, P, decomp, transform, shape, p1, p2, batch, comm_method=P2P, send_method=SYNC, prec=None):
    """dry batched plan: (rc, message, comm, plan)"""
    comm = C.c_void_p()
    check(lib().dfft_comm_create_dry(rank, P, C.byref(comm)))
    cfg = _lib.dfft_config(1, 0, comm_method, send_method, None, comm_method, send_method)
    plan = C.c_void_p()
    rc = lib().dfft_plan_create_batched(comm, C.byref(cfg), decomp, dfft.F64 if prec is None else prec, transform, shape[0], shape[1], shape[2],
                                        p1, p2, batch, 1, C.byref(plan))
    return rc, (lib().dfft_last_error_string() or b"").decode(), comm, plan


def describe_batched(rank, P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, batch, prec=None):
    rc, msg, comm, plan = create(rank, P, decomp, transform, shape, p1, p2, batch, comm_method, send_method, prec)
    assert rc == 0, msg
    need = C.c_size_t()
    check(lib().dfft_plan_describe(plan, inverse, d, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib().dfft_plan_describe(plan, inverse, d, buf, need.value, C.byref(need)))
    assert lib().dfft_get_batch(plan) == batch
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(comm)
    return json.loads(buf.value.decode())


def run_batched(P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, batch, prec=None):
    """Replays a batched exec on every rank; returns the worst rel-L2 error over all fields and ranks."""
    nx, ny, nz = shape
    c2c = transform == dfft.C2C
    scheds = [describe_batched(r, P, decomp, transform, shape, p1, p2, comm_method, send_method, inverse, d, batch, prec) for r in range(P)]
    es = scheds[0]["esize"]
    if batch > 1:
        assert all(s["batch"] == batch for s in scheds)
    lay = lambda r, w: dfft.layout(decomp, transform, nx, ny, nz, p1, p2, r, w)
    xs, specs = [], []
    for f in range(batch):  # a distinct input per field
        x = O.complex_input(shape, seed=1234 + f) if c2c else O.real_input(shape, seed=1234 + f)
        xs.append(x)
        specs.append(O.fft_c2c(x, d) if c2c else O.fft_r2c(x, d))
    mem = Memory(es)
    for r in range(P):
        for s_ in range(scheds[r]["nslots"]):
            mem.add(scheds[r]["slots"][s_][r], scheds[r]["slot_bytes"] // es)
    uin, uout, fin, fout = [], [], [], []  # user buffers and per-field sizes (complex units) per rank
    for r in range(P):
        isz, ist = lay(r, 0)
        osz, ost = lay(r, d)
        nin, nout = int(np.prod(isz)), int(np.prod(osz))
        if not c2c:
            nin //= 2  # reals, two per complex unit
        fi, fo = (nout, nin) if inverse else (nin, nout)
        if batch > 1:
            assert (scheds[r]["field_in"], scheds[r]["field_out"]) == (fi * es, fo * es)
        fin.append(fi)
        fout.append(fo)
        a = mem.add(USER_IN + (r << 48), batch * fi)
        uout.append(mem.add(USER_OUT + (r << 48), batch * fo))  # exactly batch fields: nothing beyond the last one
        for f in range(batch):
            if not inverse:
                blk = np.ascontiguousarray(O.block(xs[f], ist, isz))
                src = blk.astype(np.complex128).ravel() if c2c else blk.ravel().view(np.complex128)
            else:
                src = np.ascontiguousarray(O.block(specs[f], ost, osz)).ravel()
            a[f * fi:(f + 1) * fi] = src
        uin.append(a)
    in_copy = [a.copy() for a in uin]
    nsteps = len(scheds[0]["steps"])
    assert all(len(s["steps"]) == nsteps for s in scheds)
    order = Ordering(scheds)
    slot_owner = {}
    for r in range(P):
        for s_ in range(scheds[r]["nslots"]):
            slot_owner[scheds[r]["slots"][s_][r]] = (r, s_)

    def owner_of(addr):
        for base, (q, s_) in slot_owner.items():
            if base <= addr < base + scheds[q]["slot_bytes"]:
                return q, s_
        return None

    last_remote_write, last_rdv = {}, [-1] * P

    def user_range(r, st, which):
        """elements of the caller's buffer `which` (1 in, 2 out) this step may touch"""
        per = fin[r] if which == 1 else fout[r]
        f = st.get("field", 0)
        return (0, batch * per) if f < 0 else (f * per, (f + 1) * per)

    def user_base(r, flag):
        return {1: USER_IN, 2: USER_OUT}[flag] + (r << 48)

    for k in range(nsteps):
        pending = []
        for r in range(P):
            st = scheds[r]["steps"][k]
            if st["type"] == 1:
                last_rdv[r] = k
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
                    pending.append((dst, do, src[so:so + peer["scount"]].copy(), q))
                continue
            N = 1 << st["log2n"]
            A0, A1, B = st["A0"], st["A1"], st["B"]
            kind = st["kind"]
            if st["in_user"] == 0:
                for seg in st["in"]["segs"]:
                    own = owner_of(seg["base"])
                    assert own is not None and own[0] == r, "passes only read local memory"
                    w = last_remote_write.get(own, -1)
                    assert w < 0 or w < last_rdv[r] <= k, f"rank {r} step {k} reads slot {own} written remotely at step {w} without a rendezvous"
            if st["out_user"] == 0:
                for seg in st["out"]["segs"]:
                    own = owner_of(seg["base"])
                    assert own is not None
                    if own[0] != r:
                        assert last_rdv[r] >= 0, f"rank {r} writes into rank {own[0]}'s slot before its entry rendezvous"
                        last_remote_write[own] = k
            ub_in = user_base(r, st["in_user"]) if st["in_user"] else None
            ub_out = user_base(r, st["out_user"]) if st["out_user"] else None
            n_in, n_out = {0: (N, N), 1: (N, N), 2: (N, N + 1), 3: (N + 1, N)}[kind]
            b_ = B if kind in (0, 1) else 1

            def touched(view, n, ub, flag):
                """(array, index, ns) per segment; user accesses are checked against the step's field"""
                out = []
                for base, ns, off in view_indices(view, A0, A1, n, b_, ub):
                    arr, o = mem.resolve(base)
                    idx = o + off
                    if ub is not None:
                        lo, hi = user_range(r, st, flag)
                        assert lo <= idx.min() and idx.max() < hi, (f"rank {r} step {k} ({st['label']}) touches caller buffer {flag} at "
                                                                    f"[{idx.min()}, {idx.max()}] outside its field [{lo}, {hi})")
                    out.append((arr, idx, ns))
                return out

            data = np.zeros((A0, A1, n_in, b_), dtype=np.complex128)
            for arr, idx, ns in touched(st["in"], n_in, ub_in, st["in_user"]):
                data[:, :, ns, :] = arr[idx]
                order.read(r, k, id(arr), arr.size, idx)
            if kind in (0, 1):
                res = np.fft.ifft(data, axis=2) * N if st["inverse"] else np.fft.fft(data, axis=2)
            elif kind == 2:
                reals = np.ascontiguousarray(data[..., 0]).view(np.float64)
                res = np.fft.rfft(reals, axis=2)[..., None]
            else:
                reals = np.fft.irfft(data[..., 0], n=2 * N, axis=2) * (2 * N)
                res = np.ascontiguousarray(reals).view(np.complex128)[..., None]
            for arr, idx, ns in touched(st["out"], n_out, ub_out, st["out_user"]):
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
        assert np.array_equal(uin[r], in_copy[r]), f"rank {r}: the input was modified"
        for f in range(batch):
            if not inverse:
                osz, ost = lay(r, d)
                got = uout[r][f * fout[r]:f * fout[r] + int(np.prod(osz))].reshape(osz)
                worst = max(worst, O.rel_l2(got, O.block(specs[f], ost, osz)))
            else:
                isz, ist = lay(r, 0)
                want = O.block(xs[f], ist, isz).astype(np.complex128 if c2c else np.float64)
                scale = float(nz * (ny if d >= 2 else 1) * (nx if d >= 3 else 1))
                seg = uout[r][f * fout[r]:(f + 1) * fout[r]]
                got = seg.reshape(isz) if c2c else seg.view(np.float64).reshape(isz)
                worst = max(worst, O.rel_l2(got, want * scale))
    return worst


CASES = [
    # P, decomp, transform, shape, p1, p2, comm, send
    (1, SL, dfft.C2C, (8, 16, 64), 1, 1, P2P, SYNC),          # blocked hand-over, one rank
    (1, SL, dfft.R2C, (4, 8, 256), 1, 1, P2P, SYNC),
    (2, SL, dfft.C2C, (8, 8, 128), 2, 1, P2P, STREAMS),       # overlapped: streams join and fork again between fields
    (4, SL, dfft.C2C, (16, 8, 64), 4, 1, A2A, SYNC),
    (8, SL, dfft.R2C, (16, 8, 64), 8, 1, P2P, STREAMS),       # overlapped + blocked + tail column
    (4, SL, dfft.R2C, (8, 16, 128), 4, 1, P2P, SYNC),         # blocked + tail (Nzc = 65)
    (4, ZY, dfft.R2C, (8, 4, 32), 4, 1, P2P, SYNC),
    (4, ZY, dfft.C2C, (8, 4, 16), 4, 1, A2A, SYNC),
    (8, PE, dfft.R2C, (8, 16, 32), 2, 4, P2P, SYNC),
    (8, PE, dfft.C2C, (16, 8, 16), 4, 2, A2A, SYNC),
    (4, PE, dfft.C2C, (8, 8, 128), 2, 2, P2P, STREAMS),       # overlapped pencil forward
]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES)
@pytest.mark.parametrize("inverse", [0, 1])
def test_batched_schedules(P, decomp, transform, shape, p1, p2, comm, send, inverse):
    assert run_batched(P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, 3) < 1e-12


@pytest.mark.parametrize("d", [1, 2])
@pytest.mark.parametrize("inverse", [0, 1])
@pytest.mark.parametrize("comm", [P2P, A2A])
def test_batched_partial_schedules(d, inverse, comm):
    assert run_batched(8, PE, dfft.R2C, (8, 16, 32), 2, 4, comm, SYNC, inverse, d, 2) < 1e-12
    assert run_batched(4, PE, dfft.C2C, (8, 8, 16), 2, 2, comm, SYNC, inverse, d, 3) < 1e-12


def test_batched_overlapped_pencil_inverse(monkeypatch):
    """the overlapped pencil inverse (selected by dfft_plan_tune, built directly with DFFT_PENCIL_OVERLAP=2)"""
    monkeypatch.setenv("DFFT_PENCIL_OVERLAP", "2")
    for inverse in (0, 1):
        assert run_batched(4, PE, dfft.R2C, (8, 16, 128), 2, 2, P2P, STREAMS, inverse, 3, 2) < 1e-12


@pytest.mark.parametrize("shape,batch,prec", [((32, 32, 32), 3, dfft.F64), ((64, 64, 64), 2, dfft.F64), ((32, 32, 32), 2, dfft.F32)])
@pytest.mark.parametrize("inverse", [0, 1])
def test_batched_stage_replay(shape, batch, prec, inverse):
    """the one-launch stage, listed as its three views over all fields, against the oracle"""
    sc = describe_batched(0, 1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec)
    assert [s["field"] for s in sc["steps"]] == [-1, -1, -1]
    assert run_batched(1, SL, dfft.C2C, shape, 1, 1, P2P, SYNC, inverse, 3, batch, prec) < 1e-12


def _labels(shape, batch, inverse=0, prec=dfft.F64, transform=dfft.C2C, P=1):
    sc = describe_batched(0, P, SL, transform, shape, P, 1, P2P, SYNC, inverse, 3, batch, prec)
    return [s["label"] for s in sc["steps"]]


def test_selection_of_the_batched_stage():
    """one launch for two or more cubic 32^3 / 64^3 complex fields on one rank, in both precisions; the per-field schedule
    otherwise"""
    one = ["batched pass: z lines", "batched pass: y lines", "batched pass: x lines"]
    for n in (32, 64):
        for prec in (dfft.F64, dfft.F32):
            assert _labels((n, n, n), 2, 0, prec) == one
            assert _labels((n, n, n), 64, 1, prec) == one[::-1]
            assert _labels((n, n, n), 1, 0, prec) == ["z pass", "y pass", "x pass"]
    per_field = lambda labels, b: labels == ["z pass", "y pass", "x pass"] * b
    assert per_field(_labels((128, 128, 128), 2), 2)      # larger fields
    assert per_field(_labels((16, 16, 16), 2), 2)         # length not instantiated
    assert per_field(_labels((64, 64, 32), 2), 2)         # not cubic
    assert _labels((64, 64, 64), 2, transform=dfft.R2C)[0] == "z pass (R2C)"
    assert "batched pass" not in " ".join(_labels((64, 64, 64), 2, P=2))
    sc = describe_batched(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, P2P, SYNC, 0, 2, 2)  # partial transforms: per field
    assert [s["field"] for s in sc["steps"]] == [0, 0, 1, 1]


@pytest.mark.parametrize("P,decomp,transform,shape,p1,p2,comm,send", CASES + [(1, SL, dfft.C2C, (64, 64, 64), 1, 1, P2P, SYNC)])
def test_batch_one_is_the_unbatched_plan(P, decomp, transform, shape, p1, p2, comm, send):
    """dfft_plan_create_batched(batch = 1) describes byte for byte the schedules of dfft_plan_create"""
    for inverse in (0, 1):
        a = describe(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, 3)
        b = describe_batched(0, P, decomp, transform, shape, p1, p2, comm, send, inverse, 3, 1)
        assert json.dumps(a) == json.dumps(b)


def test_batch_argument_validation():
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, 0)
    assert rc == -1 and "batch" in msg
    lib().dfft_comm_destroy(comm)
    field = 64 ** 3 * 16
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, SIZE_MAX // field + 1)
    assert rc == -1 and "overflow" in msg
    lib().dfft_comm_destroy(comm)
    rc, msg, comm, plan = create(0, 1, SL, dfft.C2C, (64, 64, 64), 1, 1, SIZE_MAX // field)
    assert rc == 0, msg
    assert lib().dfft_get_batch(plan) == SIZE_MAX // field
    lib().dfft_plan_destroy(plan)
    lib().dfft_comm_destroy(comm)
    # R2C: the widest buffer is the complex side of the partial transforms
    rc, msg, comm, plan = create(0, 1, SL, dfft.R2C, (64, 64, 64), 1, 1, SIZE_MAX // (64 * 64 * 33 * 16) + 1)
    assert rc == -1 and "overflow" in msg
    lib().dfft_comm_destroy(comm)
    assert lib().dfft_get_batch(None) == 0


def test_work_list():
    """the field-ordered work list of the batched stage and the launch decoding of a captured / replayed launch"""
    with tempfile.TemporaryDirectory() as td:
        exe = os.path.join(td, "batch_order_test")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(HERE, "batch_order_test.cpp")], check=True)
        r = subprocess.run([exe], capture_output=True, text=True)
        assert r.returncode == 0 and "fails=0" in r.stdout, r.stdout[-2000:]
