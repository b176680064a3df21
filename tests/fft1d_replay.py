"""Replays of 1D plans (dfft_plan_create_1d) through the shared engines: step_replay's CPU interpreter and, on one GPU, the
real pass kernels through dfft_debug_run_step with gpu_replay's buffers.

A 1D plan of an n-point signal is the slab plan of its grid (N1, N2, N3): a step_replay.Plan with that shape, together with
n.  The CPU replay applies each twiddled pass's twiddle as the kernels do, from the "tw" the step list gives it: point p of
line (a0, a1) times W_n^(p (line0 + a0 + c1 a1) mul mod n), forward on the values the pass loads, inverse the conjugate on
the values it stores.  The "transpose" copy passes move a rank's x-slab to and from the y-slabs."""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager

import numpy as np

import step_replay as R
import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib


def create(p, n, factors, rank, comm=None):
    """rank's 1D plan of n points on the grid p.shape (factors None: the library's), on a geometry-only communicator when
    comm is None: (rc, message, comm, plan)"""
    c = comm
    if c is None:
        c = C.c_void_p()
        check(lib().dfft_comm_create_dry(rank, p.P, C.byref(c)))
    cfg = _lib.dfft_config(1, 0, p.comm, p.send, None, p.comm, p.send)
    plan = C.c_void_p()
    f = None if factors is None else (C.c_size_t * 3)(*factors)
    rc = lib().dfft_plan_create_1d(c, C.byref(cfg), p.prec, n, f, C.byref(plan))
    return rc, (lib().dfft_last_error_string() or b"").decode(), c, plan


def factors_of(plan):
    f = (C.c_size_t * 3)()
    check(lib().dfft_plan_get_1d_factors(plan, f))
    return tuple(int(v) for v in f)


def plan_of(P, n, factors=None, prec=dfft.F64, comm=0, scale=None):
    """the step_replay.Plan of the 1D plan (factors None: the library's choice)"""
    if factors is None:
        rc, msg, c, plan = create(R.Plan(P, dfft.SLAB_ZY_THEN_X, (0, 0, 0), prec=prec, comm=comm), n, None, 0)
        assert rc == 0, msg
        factors = factors_of(plan)
        lib().dfft_plan_destroy(plan)
        lib().dfft_comm_destroy(c)
    return R.Plan(P, dfft.SLAB_ZY_THEN_X, tuple(factors), prec=prec, comm=comm, scale=scale)


@contextmanager
def dry_plans(p, n, ranks=None):
    """the dry 1D plans of p's ranks (all of them when None), the scale set: a list of handles, destroyed on exit"""
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


def scrambled(X, shape):
    """the scrambled array [k1][k2][k3] = X[k1 + N1 k2 + N1 N2 k3] of a spectrum X"""
    n1, n2, n3 = shape
    return np.asarray(X).reshape(n3, n2, n1).transpose(2, 1, 0)


def natural(Y):
    """the spectrum X of a scrambled array (scrambled's inverse)"""
    return np.asarray(Y).transpose(2, 1, 0).ravel()


def reference(x, inverse):
    """forward: the scrambled DFT of the signal grid x [N1][N2][N3]; inverse: the signal grid of the unnormalised inverse
    DFT of the scrambled spectrum x"""
    if not inverse:
        return scrambled(np.fft.fft(np.asarray(x).ravel()), x.shape)
    n = x.size
    return (np.fft.ifft(natural(x)) * n).reshape(x.shape)


def twiddle(st, n, A0, A1, ns, conj=False):
    """[a0, a1, p, 1] twiddles of the lines (a0, a1) at points ns of twiddled pass st"""
    line0, c1, mul = st["tw"]
    line = (line0 + np.arange(A0, dtype=np.int64)[:, None] + c1 * np.arange(A1, dtype=np.int64)[None, :]) * mul
    m = (np.asarray(ns, dtype=np.int64)[None, None, :] * (line[:, :, None] % n)) % n
    w = np.exp(-2j * np.pi * m.astype(np.float64) / n)
    return (np.conj(w) if conj else w)[..., None]


class _Replay(R._Replay):
    """the shared engine with the twiddles of the y and z passes; conj=False plants an unconjugated inverse twiddle"""

    def __init__(self, p, n, scheds, inverse, conj=True):
        super().__init__(p, scheds, inverse, 3)
        self.n, self.conj, self.out_ns = n, conj, None
        assert all(sc["signal"] == n for sc in scheds)

    def check_kind(self, r, k, st, N):
        if st["kind"] == 7 and st["label"] == "transpose":  # the x-slab <-> y-slab copies of multi-rank schedules
            assert self.p.P > 1 and st["n"] == self.p.shape[1] and "twiddle" not in st, f"rank {r} step {k}"
            return
        assert st["kind"] in (0, 1), f"rank {r} step {k} ({st['label']}): 1D plans run C2C passes"
        assert ("twiddle" in st) == (st["label"] in ("y pass", "z pass")), f"rank {r} step {k} ({st['label']}): twiddle"
        super().check_kind(r, k, st, N)

    def access(self, r, k, st, which, n, b, real):
        acc = super().access(r, k, st, which, n, b, real)
        if "twiddle" not in st:
            return acc
        if which == "in" and not st["inverse"]:  # forward: the pass loads twiddled values
            out = []
            for arr, tgt, idx, cidx, ns in acc:
                tw = tgt.copy()
                tw[idx] = tgt[idx] * twiddle(st, self.n, st["A0"], st["A1"], ns)
                out.append((arr, tw, idx, cidx, ns))
            return out
        if which == "out" and st["inverse"]:
            self.out_ns = [ns for *_, ns in acc]
        return acc

    def run_pass(self, r, k, st, pending):
        start = len(pending)
        self.out_ns = None
        super().run_pass(r, k, st, pending)
        if self.out_ns is not None:  # inverse: one store per segment of the output view, in view order
            assert len(pending) - start == len(self.out_ns)
            for i, ns in zip(range(start, len(pending)), self.out_ns):
                arr, tgt, idx, cidx, val, who = pending[i]
                pending[i] = (arr, tgt, idx, cidx, val * twiddle(st, self.n, st["A0"], st["A1"], ns, self.conj), who)


def replay(p, n, inverse, x, scheds=None, mutate=None, conj=True):
    """the global output [1][N1][N2][N3] of the 1D plan on the global input grid x [N1][N2][N3]"""
    if scheds is None:
        scheds = schedules(p, n, inverse)
    if mutate:
        mutate(scheds)
    return R.assemble(_Replay(p, n, scheds, inverse, conj).run(x[None]))


def gpu_output(p, n, inverse, x):
    """The global output [1][N1][N2][N3] of the 1D plan on x, every rank's steps run in lock step on one GPU as
    gpu_replay.replay runs them: rendezvous are no-ops, all-to-all steps device copies between the ranks' staging slots, pass
    steps dfft_debug_run_step.  Checks that no output element is left unwritten and that the inputs are unchanged."""
    import gpu_replay as G
    import torch

    with dry_plans(p, n) as plans:
        scheds = [R.schedule(p, plan, inverse, 3) for plan in plans]
        sc0 = scheds[0]
        es, work_bytes = sc0["esize"], sc0["nslots"] * sc0["slot_bytes"]
        work = [G.nan_buffer(work_bytes) for _ in range(p.P)]
        bufs = [G.caller_buffers(p, sc, inverse, 3, x[None]) for sc in scheds]
        for k in range(len(sc0["steps"])):
            for r in range(p.P):
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
    got = R.assemble(outs)
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements were never written"
    return got
