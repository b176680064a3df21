"""The CPU replay of step_replay.py for plans with strides (dfft_plan_set_strides).

step_replay's engine (through box_replay's, so that box plans with strides replay too) runs these step lists unchanged.
Only the caller's buffers differ: on a side with strides each rank's block lies inside a larger array, `halo` ghost layers
on every side of it plus `gap` elements between fields, which the describe reports as "in_strides" / "out_strides".  The
ghost elements hold a poison value, every access of a pass to a caller buffer must land inside the block (a read or a
store of a ghost element fails the replay at that step), and after the exec every ghost element still holds the poison."""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import dataclass

import numpy as np

import box_replay as B
import step_replay as R
from distributedfft_b200 import R2C
from distributedfft_b200._lib import check, lib
from step_replay import USER_IN, USER_OUT, describe_raw, layouts

POISON = -3.25e300 + 7.5e299j  # every ghost element of the caller's arrays


@dataclass(frozen=True)
class Plan(B.Plan):
    """box_replay.Plan whose sides `embed` ("in", "out" or "both": the physical side, the output of d = 3) are embedded:
    `halo` ghost layers around each rank's block, `gap` more elements between fields (both in the side's elements; even on
    the real side of R2C / C2R, whose pairs of reals must stay aligned)."""
    embed: str = "both"
    halo: int = 2
    gap: int = 0


def strides(size, halo, gap):
    """{field, x, y} of a block of `size` inside its ghost layers"""
    y = size[2] + 2 * halo
    x = (size[1] + 2 * halo) * y
    return (size[0] + 2 * halo) * x + gap, x, y


def create(p, rank):
    """rank's dry plan of p with its strides, before the other setters: (rc, message, comm, plan)"""
    rc, msg, c, plan = B.create(p, rank)
    if rc != 0 or not p.embed:
        return rc, msg, c, plan
    sides = []
    for fn, name in ((lib().dfft_get_in_size, "in"), (lib().dfft_get_out_size, "out")):
        s = (C.c_size_t * 3)()
        check(fn(plan, s))
        sides.append((C.c_longlong * 3)(*strides(list(s), p.halo, p.gap)) if p.embed in (name, "both") else None)
    rc = lib().dfft_plan_set_strides(plan, *sides)
    return rc, (lib().dfft_last_error_string() or b"").decode(), c, plan


def _with_plan(p, rank, fn):
    rc, msg, c, plan = create(p, rank)
    assert rc == 0, msg
    try:
        if p.axes is not None:
            check(lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(*p.axes)))
        if p.scale is not None:
            check(lib().dfft_plan_set_scale(plan, *p.scale))
        return fn(plan)
    finally:
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)


def describe_text(p, rank, inverse, d):
    return _with_plan(p, rank, lambda plan: describe_raw(plan, inverse, d))


def describe(p, rank, inverse, d):
    """step_replay.describe of a plan with strides"""
    def parse(plan):
        assert lib().dfft_get_batch(plan) == p.fields
        sc = json.loads(describe_raw(plan, inverse, d))
        sc["domain_bytes"] = lib().dfft_get_domain_size(plan)
        sc["work_bytes"] = lib().dfft_get_work_size_device(plan)
        sc["layouts"] = layouts(plan)
        return sc
    return _with_plan(p, rank, parse)


class EmbeddedSide(R.Side):
    """R.Side of a caller buffer with strides (in the side's elements, reals on the real side of R2C / C2R): field f's block
    starts `lead` elements into the buffer, behind the ghost layers of field 0"""

    def __init__(self, p, sc, which, pairs, es, st):
        super().__init__(p, sc, which, pairs, es)
        unit = 2 if pairs else 1  # the buffer counts pairs of reals on the real side of R2C / C2R
        assert all(v % unit == 0 for v in st) and p.halo * (st[1] + st[2] + 1) % unit == 0, (st, p.halo)
        self.field, self.sx, self.sy = (v // unit for v in st)
        self.lead = p.halo * (st[1] + st[2] + 1) // unit

    def index(self, f):
        n0, n1, _ = self.size
        i = np.arange(n0)[:, None, None] * self.sx + np.arange(n1)[None, :, None] * self.sy + np.arange(self.row)[None, None, :]
        return (self.lead + f * self.field + i).ravel()


class _EmbedReplay(B._BoxReplay):
    def __init__(self, p, scheds, inverse, d):
        """step_replay's set-up of an out-of-place exec, with the caller's arrays of the embedded sides"""
        self.p, self.scheds, self.inverse, self.d = p, scheds, inverse, d
        sc0 = scheds[0]
        self.real = "r2r" in sc0
        self.es = es = sc0["esize"]
        self.r2c = p.transform == R2C and not self.real
        self.mem = R.Memory(es, np.float64 if self.real else np.complex128)
        self.owner = {}
        for r, sc in enumerate(scheds):
            assert not sc.get("inplace", False)
            for s in range(sc["nslots"]):
                self.owner[id(self.mem.add(sc["slots"][s][r], sc["slot_bytes"] // es))] = (r, s)
        src_w, dst_w = (d, 0) if inverse else (0, d)
        poison = POISON.real if self.real else POISON
        self.sides, self.bufs, self.pads, self.masks = [], [], [], []
        for r, sc in enumerate(scheds):
            sides, bufs, masks = {}, {}, {}
            for user, w, base in ((1, src_w, USER_IN), (2, dst_w, USER_OUT)):
                pairs = self.r2c and w == 0
                st = sc.get("in_strides") if w == 0 else sc.get("out_strides") if w == 3 else None
                if st is None:
                    side = R.Side(p, sc, w, pairs, es)
                    bufs[user] = self.mem.add(base + (r << 48), max(p.fields * side.field, 1))
                else:
                    side = EmbeddedSide(p, sc, w, pairs, es, st)
                    buf = self.mem.add(base + (r << 48) - side.lead * es, max(p.fields * side.field, 1))
                    mask = np.zeros(buf.size, dtype=bool)
                    for f in range(p.fields):
                        mask[side.index(f)] = True
                    buf[~mask] = poison
                    bufs[user], masks[user] = buf, mask
                if "field_in" in sc:
                    assert sc["field_in" if user == 1 else "field_out"] == side.field * es, (sc["field_in"], sc["field_out"], side.field)
                sides[user] = side
            self.sides.append(sides)
            self.bufs.append(bufs)
            self.masks.append(masks)
            self.pads.append(None)
        self.poison = poison
        self.scaled = any("scale" in st for sc in scheds for st in sc["steps"])
        self.counts = {}

    def access(self, r, k, st, which, n, b, real):
        """box_replay's access, where a caller buffer with strides is touched inside the blocks only"""
        out = super().access(r, k, st, which, n, b, real)
        user = st[which + "_user"]
        mask = self.masks[r].get(user) if user else None
        if mask is not None:
            for arr, _, _, cidx, _ in out:
                bad = ~mask[cidx]
                assert not bad.any(), (f"rank {r} step {k} ({st['label']}) {'reads' if which == 'in' else 'stores into'} "
                                       f"{int(bad.sum())} ghost elements of caller buffer {user}")
        return out

    def run(self, x):
        outs = super().run(x)
        for r in range(self.p.P):
            for user, mask in self.masks[r].items():
                assert (self.bufs[r][user][~mask] == self.poison).all(), f"rank {r}: a ghost element of caller buffer {user} changed"
        return outs


def replay(p, inverse, d, x, scheds=None, mutate=None):
    """step_replay.replay of a plan with strides: [field][rank] (start of the output block, output block)"""
    scheds = scheds or [describe(p, r, inverse, d) for r in range(p.P)]
    if mutate:
        mutate(scheds)
    return _EmbedReplay(p, scheds, inverse, d).run(x)


error = R.error
