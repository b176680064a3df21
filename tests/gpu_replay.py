"""One lock-step replay of every rank's step list on one GPU, with the real pass kernels.

The GPU counterpart of step_replay.py's engine, fed by the same step_replay.Plan: step_replay.dry_plans opens the
geometry-only plans of all P ranks, every rank gets its own work area and caller buffers (filled with 0xFF bytes, a NaN in
f32 and f64), and the ranks run in lock step: rendezvous are no-ops (the lock step orders everything), all-to-all steps are
device copies between the ranks' staging slots, and pass steps run through dfft_debug_run_step.  The caller buffers
follow step_replay.Side, so natural layouts, boxes, strides with their ghost layers, the padded real rows of in-place
R2C / C2R plans, interleaved components and batches all take one geometry.  Pruned plans come from the same creator, and
the 4-byte pairs of 16-bit plans move as uint32 elements.

`output` checks what holds for every plan: no output element is still NaN; out of place, the caller's input buffers are
unchanged byte for byte, ghosts included; every ghost byte of a strided output side is still 0xFF; and a second run with
the ranks of each step in descending order gives the same bits (a same-step hazard between ranks shows up there)."""
import ctypes as C

import numpy as np
import torch

import step_replay as R
from distributedfft_b200._lib import lib
from step_replay import assemble

SLOT_SHIFT = 44  # synthetic slot address of rank r: ((r + 1) << 44) + offset into its work area


def work_offset(addr):
    """the offset of a slot address in its rank's work area"""
    return addr & ((1 << SLOT_SHIFT) - 1)


def nan_buffer(nbytes):
    return torch.full((max(nbytes, 1),), 0xFF, dtype=torch.uint8, device="cuda")  # 0xFF..: NaN in f32 and f64


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def element_type(sc):
    """the numpy type of the elements the passes of step list sc address: real for R2R plans, else complex, and uint32 for
    the 4-byte complex elements of 16-bit plans (numpy has no complex type of two 16-bit numbers)"""
    if sc["esize"] == 4 and "r2r" not in sc:
        return np.dtype(np.uint32)
    return np.dtype(("f" if "r2r" in sc else "c") + str(sc["esize"]))


def caller_buffers(p, sc, inverse, d, x):
    """(input side, output side, input buffer, output buffer, input bytes as uploaded) of one rank: buffers of 0xFF bytes,
    the rank's blocks of x ([field][x, y, z] (+ [c])) in the input; one buffer for both sides in place"""
    dt = element_type(sc)
    i, o = R.sides(p, sc, inverse, d, dt.itemsize)
    host = np.full(i.total * dt.itemsize, 0xFF, dtype=np.uint8)
    for f in range(p.fields):
        i.put(host.view(dt), f, R.block(x[f], i.start, i.size))
    bi = torch.from_numpy(host).cuda()
    return i, o, bi, bi if p.inplace else nan_buffer(o.total * dt.itemsize), host


def run_step(plan, inverse, d, field, step, work, work_bytes, out, out_bytes, inp, in_bytes):
    """dfft_debug_run_step on torch buffers: its return code"""
    ptrs = (C.c_void_p * len(work))(*[w.data_ptr() for w in work])
    return lib().dfft_debug_run_step(plan, inverse, d, field, step, ptrs, work_bytes, out.data_ptr(), out_bytes, inp.data_ptr(), in_bytes,
                                     torch.cuda.current_stream().cuda_stream)


def replay(p, inverse, d, x, descending=False, skip=None, work_of=None):
    """Runs every rank's steps of plan p in lock step on x, the global input of the direction: [field][x, y, z] (+ [c]).
    descending: the ranks of each step in descending order; skip = (rank, step): a pass not run; work_of(rank, work): the
    work areas rank's passes see.  Checks the inputs (out of place) and the output ghosts; returns [field][rank] (start of
    the output block, output block), as step_replay.replay does."""
    with R.dry_plans(p) as plans:
        scheds = [R.schedule(p, plan, inverse, d) for plan in plans]
        sc0 = scheds[0]
        es, nslots, slot_bytes = sc0["esize"], sc0["nslots"], sc0["slot_bytes"]
        assert all(sc["nslots"] == nslots and sc["slot_bytes"] == slot_bytes for sc in scheds)
        work_bytes = nslots * slot_bytes
        work = [nan_buffer(work_bytes) for _ in range(p.P)]
        bufs = [caller_buffers(p, sc, inverse, d, x) for sc in scheds]
        items = len(sc0["steps"])
        assert all(len(sc["steps"]) == items for sc in scheds)
        per = items // p.fields
        for k in range(items):
            for r in reversed(range(p.P)) if descending else range(p.P):
                st = scheds[r]["steps"][k]
                if st["type"] == 1:
                    continue  # rendezvous: the lock step orders everything
                if st["type"] == 2:  # all-to-all-v between staging slots
                    sb = work_offset(scheds[r]["slots"][st["send_slot"]][r])
                    for peer in st["peers"]:
                        q = peer["rank"]
                        rb = work_offset(scheds[q]["slots"][st["recv_slot"]][q])
                        mine = [pp for pp in scheds[q]["steps"][k]["peers"] if pp["rank"] == r][0]
                        n = peer["scount"] * es
                        so, ro = sb + peer["soff"] * es, rb + mine["roff"] * es
                        work[q][ro:ro + n].copy_(work[r][so:so + n])
                    continue
                if skip == (r, k):
                    continue
                i, o, bi, bo, _ = bufs[r]
                inp, out = bi[i.lead * es:], bo[o.lead * es:]  # a buffer with strides: the passes take its first block element
                rc = run_step(plans[r], inverse, d, k // per, k % per, work_of(r, work) if work_of else work, work_bytes, out, out.numel(),
                              inp, inp.numel())
                assert rc == 0, f"rank {r} step {k} ({st['label']}): {(lib().dfft_last_error_string() or b'').decode()}"
        torch.cuda.synchronize()
    outs = [[] for _ in range(p.fields)]
    for r, ((i, o, bi, bo, host), sc) in enumerate(zip(bufs, scheds)):
        if not p.inplace:
            assert np.array_equal(bi.cpu().numpy(), host), f"rank {r}: the input buffer changed"
        got = bo.cpu().numpy()
        if o.strided:
            ghost = np.ones(o.total, dtype=bool)
            for f in range(p.fields):
                ghost[o.index(f)] = False
            assert (got.reshape(-1, es)[ghost] == 0xFF).all(), f"rank {r}: an output ghost element was written"
        for f in range(p.fields):
            outs[f].append((o.start, o.get(got.view(element_type(sc)), f)))
    return outs


def output(p, inverse, d, x):
    """the global output (field, ...) of plan p on x, after the checks every plan gets (see the module's description)"""
    got = assemble(replay(p, inverse, d, x))
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements were never written"
    again = assemble(replay(p, inverse, d, x, descending=True))
    assert same_bits(again, got), "the result depends on the order of the ranks within a step"
    return got
