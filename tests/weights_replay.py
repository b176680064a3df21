"""Replays of weighted plans (dfft_plan_set_weights) through the shared engines: step_replay's CPU interpreter and, on one
GPU, the real pass kernels through dfft_debug_run_step with gpu_replay's buffers.

A weighted plan is a step_replay.Plan and its (wx, wy, wz) tables, each None or one value per point of the axis's spectral
view.  numpy tables give the geometry-only plans stand-in pointers, which they never dereference; torch CUDA tensors give
their device pointers, which the GPU replay's kernels read.  The CPU replay multiplies the spectral side of every pass the
step list marks "weighted" by the table of its "axis", at the index of each value in that side's view: forward the
values the pass stores, inverse the values it loads."""
from __future__ import annotations

import ctypes as C
from contextlib import contextmanager

import numpy as np

import step_replay as R
from distributedfft_b200._lib import check, lib

STANDIN = 1 << 40  # stand-in table pointers of geometry-only plans (axis a: + a << 20)


@contextmanager
def dry_plans(p, weights, ranks=None):
    """step_replay.dry_plans with the tables set on every plan, before anything builds a schedule"""
    given = [None if w is None else w.data_ptr() if hasattr(w, "data_ptr") else STANDIN + (a << 20) for a, w in enumerate(weights)]
    with R.dry_plans(p, ranks) as plans:
        for plan in plans:
            check(lib().dfft_plan_set_weights(plan, (C.c_void_p * 3)(*given)))
        yield plans


def describe(p, weights, rank, inverse, d):
    """rank's parsed step list of the weighted plan (step_replay.schedule)"""
    with dry_plans(p, weights, [rank]) as (plan,):
        return R.schedule(p, plan, inverse, d)


def replay(p, weights, inverse, d, x, scheds=None):
    """step_replay.replay of the weighted plan"""
    if scheds is None:
        with dry_plans(p, weights) as plans:
            scheds = [R.schedule(p, plan, inverse, d) for plan in plans]
    return _Replay(p, weights, scheds, inverse, d).run(x)


class _Replay(R._Replay):
    """the shared engine, its passes' spectral sides multiplied by the tables"""

    def __init__(self, p, weights, scheds, inverse, d):
        super().__init__(p, scheds, inverse, d)
        self.weights = [None if w is None else np.asarray(w) for w in weights]
        self.out_ns = None

    def table(self, r, k, st):
        """the table pass st multiplies by, None for none; every FFT pass of a weighted plan is marked"""
        assert ("weighted" in st) == (st["kind"] not in (6, 7)), f"rank {r} step {k} ({st['label']}): weighted pass"
        return self.weights[st["axis"]] if "weighted" in st else None

    def access(self, r, k, st, which, n, b, real):
        acc = super().access(r, k, st, which, n, b, real)
        w = self.table(r, k, st)
        if w is None:
            return acc
        if which == "in" and st["inverse"]:  # the pass loads weighted values: a weighted copy of each array it reads
            out = []
            for arr, tgt, idx, cidx, ns in acc:
                tw = tgt.copy()
                tw[idx] = tgt[idx] * w[ns][None, None, :, None]
                out.append((arr, tw, idx, cidx, ns))
            return out
        if which == "out" and not st["inverse"]:
            self.out_ns = [ns for *_, ns in acc]
        return acc

    def run_pass(self, r, k, st, pending):
        start = len(pending)
        self.out_ns = None
        super().run_pass(r, k, st, pending)
        if self.out_ns is not None:  # forward: run_pass queues one store per segment of its output view, in view order
            w = self.table(r, k, st)
            assert len(pending) - start == len(self.out_ns)
            for i, ns in zip(range(start, len(pending)), self.out_ns):
                arr, tgt, idx, cidx, val, who = pending[i]
                pending[i] = (arr, tgt, idx, cidx, val * w[ns][None, None, :, None], who)


def gpu_output(p, weights, inverse, d, x):
    """The global output (field, ...) of the weighted plan p (torch CUDA tables) on x, every rank's steps run in lock step on
    one GPU as gpu_replay.replay runs them: rendezvous are no-ops, all-to-all steps device copies between the ranks'
    staging slots, pass steps dfft_debug_run_step.  Checks that no output element is left unwritten and, out of place,
    that the inputs are unchanged."""
    import gpu_replay as G
    import torch

    with dry_plans(p, weights) as plans:
        scheds = [R.schedule(p, plan, inverse, d) for plan in plans]
        sc0 = scheds[0]
        es, work_bytes = sc0["esize"], sc0["nslots"] * sc0["slot_bytes"]
        work = [G.nan_buffer(work_bytes) for _ in range(p.P)]
        bufs = [G.caller_buffers(p, sc, inverse, d, x) for sc in scheds]
        items = len(sc0["steps"])
        per = items // p.fields
        for k in range(items):
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
                        n = peer["scount"] * es
                        so, ro = sb + peer["soff"] * es, rb + mine["roff"] * es
                        work[q][ro:ro + n].copy_(work[r][so:so + n])
                    continue
                i, o, bi, bo, _ = bufs[r]
                inp, out = bi[i.lead * es:], bo[o.lead * es:]
                rc = G.run_step(plans[r], inverse, d, k // per, k % per, work, work_bytes, out, out.numel(), inp, inp.numel())
                assert rc == 0, f"rank {r} step {k} ({st['label']}): {(lib().dfft_last_error_string() or b'').decode()}"
        torch.cuda.synchronize()
    outs = [[] for _ in range(p.fields)]
    for r, ((i, o, bi, bo, host), sc) in enumerate(zip(bufs, scheds)):
        if not p.inplace:
            assert np.array_equal(bi.cpu().numpy(), host), f"rank {r}: the input buffer changed"
        got = bo.cpu().numpy()
        for f in range(p.fields):
            outs[f].append((o.start, o.get(got.view(G.element_type(sc)), f)))
    got = R.assemble(outs)
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} output elements were never written"
    return got
