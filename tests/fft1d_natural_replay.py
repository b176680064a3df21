"""Replays of natural-order 1D plans (dfft_plan_create_1d_natural) through the shared engines, extending fft1d_replay for
the transposing z pass.

The z pass of a natural-order plan runs TILED in its transposing form: its step lists "transposed": sB, the stride along b
of its row side (forward its input, inverse its output), which holds line b's point p at b sB + p; the other side is the
plain TILED view.  Its twiddle's line index is line0 + b + c1 a0 (k1 = x0 + b, k2 = a0), where the other twiddled passes
take line0 + a0 + c1 a1.  On more than one rank the "landing copy" (forward) and the "scatter copy" (inverse) move each
rank's output chunk [oz_r][N2][N1] between the caller's buffer and the landing slot, lines along k1.

The global output of a forward replay is the grid [N3][N2][N1]: flattened, numpy.fft.fft of the flattened signal."""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager

import numpy as np

import fft1d_replay as F
import step_replay as R
import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib


def create(p, n, factors, rank, comm=None):
    """rank's natural-order 1D plan of n points on the grid `factors` (None: the library's), on a geometry-only communicator
    when comm is None: (rc, message, comm, plan)"""
    c = comm
    if c is None:
        c = C.c_void_p()
        check(lib().dfft_comm_create_dry(rank, p.P, C.byref(c)))
    cfg = _lib.dfft_config(1, 0, p.comm, p.send, None, p.comm, p.send)
    plan = C.c_void_p()
    f = None if factors is None else (C.c_size_t * 3)(*factors)
    rc = lib().dfft_plan_create_1d_natural(c, C.byref(cfg), p.prec, n, f, C.byref(plan))
    return rc, (lib().dfft_last_error_string() or b"").decode(), c, plan


def plan_of(P, n, factors=None, prec=dfft.F64, comm=0, scale=None):
    """the step_replay.Plan of the natural-order plan (factors None: the library's choice)"""
    if factors is None:
        rc, msg, c, plan = create(R.Plan(P, dfft.SLAB_ZY_THEN_X, (0, 0, 0), prec=prec, comm=comm), n, None, 0)
        assert rc == 0, msg
        factors = F.factors_of(plan)
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)
    return R.Plan(P, dfft.SLAB_ZY_THEN_X, tuple(factors), prec=prec, comm=comm, scale=scale)


@contextmanager
def dry_plans(p, n, ranks=None):
    """the dry natural-order plans of p's ranks (all of them when None), the scale set, destroyed on exit"""
    made = []
    try:
        for r in range(p.P) if ranks is None else ranks:
            rc, msg, c, plan = create(p, n, p.shape, r)
            made.append((c, plan))
            assert rc == 0, msg
            R.set_options(p, plan)
        yield [plan for _, plan in made]
    finally:
        for c, plan in made:
            lib().dfft_plan_destroy(plan)
            lib().dfft_comm_destroy(c)


def schedules(p, n, inverse):
    with dry_plans(p, n) as plans:
        return [R.schedule(p, plan, inverse, 3) for plan in plans]


def reference(x, inverse):
    """forward: the spectrum of the signal grid x [N1][N2][N3] as the grid [N3][N2][N1]; inverse: the signal grid [N1][N2][N3]
    of the unnormalised inverse DFT of the natural-order spectrum x [N3][N2][N1]"""
    n = x.size
    if not inverse:
        n1, n2, n3 = x.shape
        return np.fft.fft(np.asarray(x).ravel()).reshape(n3, n2, n1)
    n3, n2, n1 = x.shape
    return (np.fft.ifft(np.asarray(x).ravel()) * n).reshape(n1, n2, n3)


def transposed_twiddle(st, n, ns, conj=False, line_b=True):
    """[a0, 1, p, b] twiddles of the transposing pass st at points ns: W_n^(p (line0 + b + c1 a0) mul mod n); line_b=False
    plants a line index without b (k1 missing)"""
    line0, c1, mul = st["tw"]
    b = np.arange(st["B"], dtype=np.int64)[None, :] if line_b else np.zeros((1, 1), dtype=np.int64)
    line = ((line0 + b + c1 * np.arange(st["A0"], dtype=np.int64)[:, None]) * mul) % n  # [a0, b]
    m = (np.asarray(ns, dtype=np.int64)[None, :, None] * line[:, None, :]) % n  # [a0, p, b]
    w = np.exp(-2j * np.pi * m.astype(np.float64) / n)[:, None, :, :]
    return np.conj(w) if conj else w


class _Replay(F._Replay):
    """fft1d_replay's engine with the transposing z pass and the natural copies; line_b=False plants a twiddle without k1"""

    def __init__(self, p, n, scheds, inverse, line_b=True):
        super().__init__(p, n, scheds, inverse)
        self.line_b = line_b
        assert all(sc.get("order") == "natural" for sc in scheds)

    def check_kind(self, r, k, st, N):
        where = f"rank {r} step {k} ({st['label']})"
        if st["label"] in ("landing copy", "scatter copy"):
            assert self.p.P > 1 and st["kind"] == 6 and st["n"] == self.p.shape[0] and st["B"] == 1 and "twiddle" not in st, where
            assert st["label"] == ("scatter copy" if self.inverse else "landing copy"), where
            return
        if "transposed" in st:
            n1, n2, n3 = self.p.shape
            assert st["label"] == "z pass" and st["kind"] == 1 and st["transposed"] == n2 * n3 and st["A1"] == 1, where
            row = st["out" if st["inverse"] else "in"]
            assert row["nseg"] == 1 and row["sN"] == 1, where
        else:
            assert st["label"] != "z pass", f"{where}: the z pass of a natural-order plan transposes"
        super().check_kind(r, k, st, N)

    def _tw(self, st, ns, conj=False):
        if "transposed" in st:
            return transposed_twiddle(st, self.n, ns, conj, self.line_b)
        return F.twiddle(st, self.n, st["A0"], st["A1"], ns, conj)

    def access(self, r, k, st, which, n, b, real):
        row = "transposed" in st and which == ("out" if st["inverse"] else "in")
        acc = R._Replay.access(self, r, k, st, which, n, 1 if row else b, real)
        if row:  # line b of the row side starts b * sB elements in
            off = np.arange(b, dtype=np.int64)[None, None, None, :] * st["transposed"]
            acc = [(arr, tgt, idx + off, cidx + off, ns) for arr, tgt, idx, cidx, ns in acc]
        if "twiddle" not in st:
            return acc
        if which == "in" and not st["inverse"]:  # forward: the pass loads twiddled values
            out = []
            for arr, tgt, idx, cidx, ns in acc:
                tw = tgt.copy()
                tw[idx] = tgt[idx] * self._tw(st, ns)
                out.append((arr, tw, idx, cidx, ns))
            return out
        if which == "out" and st["inverse"]:
            self.out_ns = [ns for *_, ns in acc]
        return acc

    def run_pass(self, r, k, st, pending):
        start = len(pending)
        self.out_ns = None
        R._Replay.run_pass(self, r, k, st, pending)
        if self.out_ns is not None:  # inverse: one store per segment of the output view, times the conjugate twiddles
            assert len(pending) - start == len(self.out_ns)
            for i, ns in zip(range(start, len(pending)), self.out_ns):
                arr, tgt, idx, cidx, val, who = pending[i]
                pending[i] = (arr, tgt, idx, cidx, val * self._tw(st, ns, conj=True), who)


def replay(p, n, inverse, x, scheds=None, mutate=None, line_b=True):
    """the global output [N3][N2][N1] (forward) or [N1][N2][N3] (inverse) of the natural-order plan on the global input x of
    the direction: the signal grid [N1][N2][N3] forward, the spectrum grid [N3][N2][N1] inverse"""
    if scheds is None:
        scheds = schedules(p, n, inverse)
    if mutate:
        mutate(scheds)
    return R.assemble(_Replay(p, n, scheds, inverse, line_b).run(x[None]))[0]


def gpu_output(p, n, inverse, x, descending=False):
    """The global output of the natural-order plan on x (as replay returns it), every rank's steps run in lock step on one
    GPU as fft1d_replay.gpu_output runs them: NaN-poisoned work areas, rendezvous as no-ops, all-to-all steps as device
    copies between the ranks' staging slots, pass steps through dfft_debug_run_step.  descending: the ranks of each step in
    descending order (gpu_replay.replay's same-step hazard check).  Checks that the inputs are unchanged and that every
    output element was written."""
    import gpu_replay as G
    import torch

    with dry_plans(p, n) as plans:
        scheds = [R.schedule(p, plan, inverse, 3) for plan in plans]
        sc0 = scheds[0]
        es, work_bytes = sc0["esize"], sc0["nslots"] * sc0["slot_bytes"]
        work = [G.nan_buffer(work_bytes) for _ in range(p.P)]
        bufs = [G.caller_buffers(p, sc, inverse, 3, x[None]) for sc in scheds]
        for k in range(len(sc0["steps"])):
            for r in reversed(range(p.P)) if descending else range(p.P):
                st = scheds[r]["steps"][k]
                if st["type"] == 1:
                    continue
                if st["type"] == 2:
                    sb = G.work_offset(scheds[r]["slots"][st["send_slot"]][r])
                    for peer in st["peers"]:
                        q = peer["rank"]
                        rb = G.work_offset(scheds[q]["slots"][st["recv_slot"]][q])
                        mine = [pp for pp in scheds[q]["steps"][k]["peers"] if pp["rank"] == r][0]
                        m = peer["scount"] * es
                        so, ro = sb + peer["soff"] * es, rb + mine["roff"] * es
                        work[q][ro:ro + m].copy_(work[r][so:so + m])
                    continue
                i, o, bi, bo, _ = bufs[r]
                inp, out = bi[i.lead * es:], bo[o.lead * es:]
                rc = G.run_step(plans[r], inverse, 3, 0, k, work, work_bytes, out, out.numel(), inp, inp.numel())
                assert rc == 0, f"rank {r} step {k} ({st['label']}): {(lib().dfft_last_error_string() or b'').decode()}"
        torch.cuda.synchronize()
    outs = [[]]
    for r, ((i, o, bi, bo, host), sc) in enumerate(zip(bufs, scheds)):
        assert np.array_equal(bi.cpu().numpy(), host), f"rank {r}: the input buffer changed"
        outs[0].append((o.start, o.get(bo.cpu().numpy().view(G.element_type(sc)), 0)))
    got = R.assemble(outs)[0]
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements were never written"
    return got
