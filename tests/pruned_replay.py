"""Pruned plans (dfft_plan_create_pruned) in the lock-step replays of step_replay.py (numpy) and gpu_replay.py (the real
kernels on one GPU).

Both engines open their dry plans through step_replay's plan creator; `plans()` lets that creator make pruned plans from
`Plan.data` and hands every other plan to it unchanged.  The CPU engine's `Replay` adds the "data" key of a pass: its
physical side (in forward, out inverse) holds line positions [0, data) only (R2C / C2R: data reals, data / 2 pairs), the
rest of the line is zero.  A pass without the key runs step_replay's own code."""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager
from dataclasses import dataclass
from unittest import mock

import numpy as np

import step_replay as R
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib


@dataclass(frozen=True)
class Plan(R.Plan):
    """step_replay's Plan with the data block of a pruned plan: (mx, my, mz), created by dfft_plan_create_pruned together
    with `spectral` (None: the whole grid).  Pruned plans have no strides, boxes or components."""
    data: tuple | None = None


_create = R.create


def create(p, rank, comm=None):
    """step_replay.create, which also makes the pruned plans of Plan.data: (rc, message, comm, plan)"""
    if getattr(p, "data", None) is None:
        return _create(p, rank, comm)
    assert p.in_boxes is None and p.out_boxes is None and p.embed is None and p.components is None and p.kinds is None and not p.inplace
    c = comm
    if c is None:
        c = C.c_void_p()
        check(lib().dfft_comm_create_dry(rank, p.P, C.byref(c)))
    cfg = C.byref(_lib.dfft_config(1, 0, p.comm, p.send, None, p.comm, p.send))
    plan = C.c_void_p()
    k = None if p.spectral is None else (C.c_size_t * 3)(*p.spectral)
    rc = lib().dfft_plan_create_pruned(c, cfg, p.decomp, p.prec, p.transform, *p.shape, (C.c_size_t * 3)(*p.data), k, p.p1, p.p2, p.fields, 1,
                                       C.byref(plan))
    return rc, (lib().dfft_last_error_string() or b"").decode(), c, plan


@contextmanager
def plans():
    """step_replay.dry_plans (and so describe, replay and gpu_replay) with pruned plans"""
    with mock.patch.object(R, "create", create):
        yield


class Replay(R._Replay):
    """the CPU engine with the "data" key of a pass, and the check that a pruned plan runs such a pass on every axis with
    M < N among its first d"""

    def run(self, x):
        self.data_holes = 0
        outs = super().run(x)
        p = self.p
        if getattr(p, "data", None) is not None and any(p.data[a] != p.shape[a] for a in (2, 1, 0)[:self.d]):
            assert self.data_holes > 0, "a pruned plan with data smaller than one of its first d axes runs no pass with a data hole"
        return outs

    def check_kind(self, r, k, st, N):
        super().check_kind(r, k, st, N)
        if "data" in st:
            kind = st["kind"]
            where = f"rank {r} step {k} ({st['label']}, kind {kind})"
            self.data_holes += 1
            assert kind in (0, 1, 2, 3) and 1 <= st["data"] < (2 * N if kind in (2, 3) else N), where
            assert kind not in (2, 3) or st["data"] % 2 == 0, where

    def run_pass(self, r, k, st, pending):
        if "data" not in st:
            return super().run_pass(r, k, st, pending)
        # step_replay's run_pass with the physical side cut to [0, data): read and zero-embedded forward, computed and
        # truncated inverse; the spectral side keeps its "keep" rule
        kind, inv = st["kind"], st["inverse"]
        N = st.get("n", 1 << st["log2n"])
        self.check_kind(r, k, st, N)
        points, real_in, real_out, math = R.PASSES[kind]
        n_in, n_out = points(N)
        b = 1 if kind in (2, 3) else st["B"]
        A0, A1 = st["A0"], st["A1"]
        keep = st.get("keep")
        phys = st["data"] // 2 if kind in (2, 3) else st["data"]
        kin = (keep if keep is not None else n_in) if inv else phys
        kout = phys if inv else (keep if keep is not None else n_out)
        reads = self.access(r, k, st, "in", kin, b, real_in)
        writes = self.access(r, k, st, "out", kout, b, real_out)
        data = np.zeros((A0, A1, kin, b), dtype=np.complex128 if not real_in else np.float64)
        for arr, tgt, idx, cidx, ns in reads:
            data[:, :, ns, :] = tgt[idx]
            self.order.read(r, k, id(arr), arr.size, cidx)
        self.check_buffer(r, k, st, reads, writes)
        self.check_bounds(r, k, st, "in", reads)
        self.check_bounds(r, k, st, "out", writes)
        if kin != n_in:
            full = np.zeros((A0, A1, n_in, b), dtype=data.dtype)
            full[:, :, (R.positions(N, kin) if kind != 3 else np.arange(kin)) if inv else np.arange(kin), :] = data
            data = full
        res = math(st, data, N)
        if kout != n_out:
            res = res[:, :, np.arange(kout) if inv else (R.positions(N, kout) if kind != 2 else np.arange(kout)), :]
        if "scale" in st:
            res = res * st["scale"]
            for arr, tgt, idx, cidx, ns in writes:
                assert st["out_user"] == 2, f"rank {r} step {k} ({st['label']}): only stores into the caller's output are scaled"
                cnt = self.counts.setdefault(id(arr), np.zeros(arr.size * 2, dtype=np.int64))
                if tgt is arr:
                    for j in range(2):
                        np.add.at(cnt, 2 * idx.ravel() + j, 1)
                else:
                    np.add.at(cnt, idx.ravel(), 1)
        for arr, tgt, idx, cidx, ns in writes:
            pending.append((arr, tgt, idx, cidx, res[:, :, ns, :], r))


def replay(p, inverse, d, x, scheds=None):
    """step_replay.replay for pruned plans (and any other)"""
    if scheds is None:
        with plans(), R.dry_plans(p) as opened:
            scheds = [R.schedule(p, plan, inverse, d) for plan in opened]
    return Replay(p, scheds, inverse, d).run(x)


def describe(p, rank, inverse, d):
    """step_replay.describe for pruned plans (and any other)"""
    with plans():
        return R.describe(p, rank, inverse, d)
