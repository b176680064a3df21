"""The CPU replay of step_replay.py for box-distributed plans (dfft_plan_create_boxes).

step_replay's engine runs these step lists unchanged, with two additions that only box plans need:
  - their reshape copies ("reshape in" / "reshape out", kind 6 over the boxes' views) are a pass kind of their own;
  - a "reshape out" step gathers its pieces from the peers' staging slots: it reads remote memory, which no other pass does.
    The happens-before check covers those reads like every other access (the rendezvous before the gather orders them
    behind the stores of the last FFT pass on every rank)."""
from __future__ import annotations

import ctypes as C
import json
from dataclasses import dataclass

import numpy as np

import step_replay as R
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from step_replay import USER_IN, USER_OUT, describe_raw, layouts, view_indices


@dataclass(frozen=True)
class Plan(R.Plan):
    """step_replay.Plan with one ((lx, ly, lz), (hx, hy, hz)) per rank of the physical (in_boxes) and the output grid
    (out_boxes); None keeps that side's natural layout.  A plan with boxes is made by dfft_plan_create_boxes."""
    in_boxes: tuple | None = None
    out_boxes: tuple | None = None


def flat(boxes):
    return None if boxes is None else (C.c_size_t * (6 * len(boxes)))(*[v for lo, hi in boxes for v in (*lo, *hi)])


def create(p, rank):
    """rank's dry plan of p, before the setters: (rc, message, comm, plan)"""
    if p.in_boxes is None and p.out_boxes is None:
        return R.create(p, rank)
    c = C.c_void_p()
    check(lib().dfft_comm_create_dry(rank, p.P, C.byref(c)))
    cfg = C.byref(_lib.dfft_config(1, 0, p.comm, p.send, None, p.comm, p.send))
    plan = C.c_void_p()
    rc = lib().dfft_plan_create_boxes(c, cfg, p.decomp, p.prec, p.transform, *p.shape, p.p1, p.p2, flat(p.in_boxes), flat(p.out_boxes),
                                      p.fields, 1, C.byref(plan))
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
    """step_replay.describe of a box plan"""
    def parse(plan):
        assert lib().dfft_get_batch(plan) == p.fields
        sc = json.loads(describe_raw(plan, inverse, d))
        sc["domain_bytes"] = lib().dfft_get_domain_size(plan)
        sc["work_bytes"] = lib().dfft_get_work_size_device(plan)
        sc["layouts"] = layouts(plan)
        return sc
    return _with_plan(p, rank, parse)


class _BoxReplay(R._Replay):
    def check_kind(self, r, k, st, N):
        if st["kind"] == 6 and st["label"].startswith("reshape"):
            where = f"rank {r} step {k} ({st['label']})"
            assert self.p.in_boxes is not None or self.p.out_boxes is not None, where
            assert "n" in st and st["log2n"] == 0 and "r2r" not in st and st["B"] == 1, where
            return
        super().check_kind(r, k, st, N)

    def access(self, r, k, st, which, n, b, real):
        """step_replay's access, where "reshape out" steps may read a peer's slot"""
        user = st[which + "_user"]
        ub = {1: USER_IN, 2: USER_IN if self.p.inplace else USER_OUT}[user] + (r << 48) if user else None
        out = []
        for base, ns, off in view_indices(st[which], st["A0"], st["A1"], n, b, ub):
            if off.size == 0:
                continue
            arr, o = self.mem.resolve(base)
            tgt, idx = (arr.view(np.float64), 2 * o + off) if real else (arr, o + off)
            cidx = idx // 2 if real else idx
            if not user:
                own = self.owner.get(id(arr))
                assert own is not None, f"rank {r} step {k} ({st['label']}): a slot view outside the slots"
                if which == "in":
                    assert own[0] == r or st["label"] == "reshape out", "passes other than the output gathers read only local memory"
                    w = self.last_remote_write.get(own, -1)
                    assert w < 0 or w < self.last_rdv[r] <= k, f"rank {r} step {k} reads slot {own} written remotely at step {w} without a rendezvous"
                elif own[0] != r:
                    assert self.last_rdv[r] >= 0, f"rank {r} writes into rank {own[0]}'s slot before its entry rendezvous"
                    self.last_remote_write[own] = k
            out.append((arr, tgt, idx, cidx, ns))
        return out


def replay(p, inverse, d, x, scheds=None, mutate=None):
    """step_replay.replay of a box plan: [field][rank] (start of the output box, output box)"""
    scheds = scheds or [describe(p, r, inverse, d) for r in range(p.P)]
    if mutate:
        mutate(scheds)
    return _BoxReplay(p, scheds, inverse, d).run(x)


error = R.error
