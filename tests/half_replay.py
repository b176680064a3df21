"""16-bit plans (DFFT_F16 / DFFT_BF16) in the lock-step replays of step_replay.py (numpy) and gpu_replay.py (the real
kernels on one GPU).

Both engines address elements of 8 or 16 bytes; a 16-bit plan's step list addresses 4-byte ones.
  - CPU: `widened` rewrites a 16-bit step list at 8 bytes per element — every byte quantity (slot size and addresses,
    caller offsets, field distances, domain and work sizes) doubled, every element count and view unchanged — so the
    numpy engine replays exactly its steps; `Replay` stores each pass's values times its "factor" and rounded to 16 bits
    (`store16`), as the kernels do.
  - GPU: `gpu_replay` runs the steps through dfft_debug_run_step, which needs only the buffers' element type: `elements`
    lets it move the 4-byte pairs as uint32 (numpy has no complex type of two 16-bit numbers)."""
from __future__ import annotations

from contextlib import contextmanager
from unittest import mock

import numpy as np

import distributedfft_b200 as dfft
import gpu_replay as G
import step_replay as R

SLOT_SHIFT = 44  # synthetic slot address of rank r: ((r + 1) << 44) + offset into its work area


def round16(v, prec):
    """v rounded to binary16 (numpy, round to nearest even) or bfloat16 (nearest even on the float32 bits), as float64"""
    v = np.asarray(v)
    if np.iscomplexobj(v):
        return round16(v.real, prec) + 1j * round16(v.imag, prec)
    if prec == dfft.F16:
        return v.astype(np.float16).astype(np.float64)
    u = v.astype(np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32)
    return u.view(np.float32).astype(np.float64)


def store16(st, res, prec):
    """what a 16-bit pass st stores of its values res: times its factor in f32, rounded once"""
    f = st.get("factor")
    if f is not None:
        res = (res.real.astype(np.float32) * np.float32(f)).astype(np.float64) + (
            1j * (res.imag.astype(np.float32) * np.float32(f)).astype(np.float64) if np.iscomplexobj(res) else 0)
    return round16(res, prec)


def widened(sc):
    """the 4-byte step list sc (step_replay.schedule) with 8 bytes per element"""
    assert sc["esize"] == 4, sc["esize"]

    def addr(b):
        if b >> SLOT_SHIFT:  # a slot: the rank bits stay, the offset into the work area doubles
            return ((b >> SLOT_SHIFT) << SLOT_SHIFT) + 2 * (b & ((1 << SLOT_SHIFT) - 1))
        return 2 * b  # an offset into the caller's buffer

    out = dict(sc, esize=8, slot_bytes=2 * sc["slot_bytes"], domain_bytes=2 * sc["domain_bytes"], work_bytes=2 * sc["work_bytes"],
               slots=[[addr(a) for a in s] for s in sc["slots"]])
    for key in ("field_in", "field_out"):
        if key in sc:
            out[key] = 2 * sc[key]
    steps = []
    for st in sc["steps"]:
        st = dict(st)
        for w in ("in", "out"):
            if w in st:
                st[w] = {**st[w], "segs": [{**g, "base": addr(g["base"])} for g in st[w]["segs"]]}
        steps.append(st)
    out["steps"] = steps
    return out


class Replay(R._Replay):
    """the CPU engine on a widened 16-bit step list, every pass's stores as store16 makes them"""

    def __init__(self, p, scheds, inverse, d):
        super().__init__(p, [widened(sc) for sc in scheds], inverse, d)

    def run_pass(self, r, k, st, pending):
        mine = []
        super().run_pass(r, k, st, mine)
        for arr, tgt, idx, cidx, val, who in mine:
            pending.append((arr, tgt, idx, cidx, store16(st, val, self.p.prec), who))


def replay(p, inverse, d, x):
    """step_replay.replay for the 16-bit plan p: [field][rank] (start of the output block, output block)"""
    with R.dry_plans(p) as plans:
        scheds = [R.schedule(p, plan, inverse, d) for plan in plans]
    return Replay(p, scheds, inverse, d).run(x)


def element_type(sc):
    """gpu_replay.element_type, with the 4-byte complex elements of 16-bit plans as uint32"""
    if sc["esize"] == 4 and "r2r" not in sc:
        return np.dtype(np.uint32)
    return np.dtype(("f" if "r2r" in sc else "c") + str(sc["esize"]))


@contextmanager
def elements():
    """gpu_replay.replay (and caller_buffers) with element_type above"""
    with mock.patch.object(G, "element_type", element_type):
        yield
