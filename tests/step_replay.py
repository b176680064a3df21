"""One CPU interpreter of the step lists dfft_plan_describe emits, for every plan form and any rank count.

dfft_comm_create_dry gives a geometry-only communicator; dfft_plan_describe returns, per rank, the exact step list the GPU
executes: every pass with its segmented input / output views (base addresses, strides, segment tables), rendezvous points
and all-to-all counts.  `replay` builds the plans of all P ranks, lays the synthetic slot and caller addresses out in numpy
arrays, executes the steps in lock step (numpy / scipy per pass, the views for all data movement) and returns every rank's
output block of every field.  On the way it checks what the step lists promise and the lock-step data flow cannot show,
each wherever it applies:
  - happens-before (Ordering): every read-after-write and write-after-read is ordered by a stream, an event or a rendezvous;
  - every rank lists as many steps, and both ends of an all-to-all agree on its counts;
  - slots: a pass reads only its own rank's slots (the "reshape out" gathers of box plans read their peers'), stores into a
    peer's slot only after its entry rendezvous, and reads a slot a peer stored into only after a later rendezvous;
  - out of place, the caller's input is left intact;
  - on a side with strides, the ghost elements around each block (poisoned) are neither read nor stored into;
  - a per-field step stays inside its field of the caller's buffers; with a scale, every output value is scaled exactly
    once, and only by stores into the caller's output;
  - a step that stores into an array it also reads stores every element from the line that reads it, or one that no other
    line reads (the passes load a line or tile completely before they store it);
  - the two listed phases of the fused z + y stage and of the batched stage, which run concurrently, touch disjoint
    planes / fields;
  - in-place R2C / C2R plans: the padding of the real rows is not read before a store, and the C2R pass never stores there;
  - every pass names a kind this module knows, with the lengths, line counts and strides that kind takes, a padded plan
    has a hole pass ("keep") wherever one of the first d axes is truncated, and a pruned plan has a data-hole pass
    ("data") wherever its data is smaller than one of the first d axes.
16-bit plans (F16 / BF16) address 4-byte elements; the replay computes in double as for every plan and rounds each pass's
stores to 16 bits, after its "factor", as the kernels do."""
from __future__ import annotations

import ctypes as C
import json
from contextlib import contextmanager
from dataclasses import dataclass

import numpy as np
import scipy.fft as sf

import distributedfft_b200 as dfft
from distributedfft_b200 import _lib
from distributedfft_b200._lib import check, lib
from oracle import dft_oracle as O

USER_IN, USER_OUT = 1 << 60, 1 << 61  # synthetic address ranges of the caller's buffers (rank r: + r << 48)
PAD = 1234.5 - 678.25j  # value of the padding of the real rows of in-place R2C / C2R plans
POISON = -3.25e300 + 7.5e299j  # every ghost element of a caller array with strides


# ---- plans ----------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Plan:
    """Everything a replayed plan can have.  The creator follows the fields: data -> dfft_plan_create_pruned, boxes ->
    dfft_plan_create_boxes, spectral -> dfft_plan_create_padded, components -> dfft_plan_create_interleaved, kinds ->
    dfft_plan_create_r2r, inplace -> dfft_plan_create_inplace, a batch -> dfft_plan_create_batched, else dfft_plan_create.
    embed, axes and scale go through their setters.

    in_boxes / out_boxes: one ((lx, ly, lz), (hx, hy, hz)) per rank of the physical and the output grid; None keeps that
    side's natural layout.  embed ("in", "out" or "both": the physical side, the output of d = 3) puts each rank's block of
    those sides inside a larger caller array: `halo` ghost layers around it, `gap` more elements between fields (both in the
    side's elements; even on the real side of R2C / C2R, whose pairs of reals must stay aligned).  data: the (mx, my, mz)
    block of a pruned plan, made together with `spectral` (None: the whole grid); pruned plans have no boxes, strides,
    components, kinds or in-place form."""
    P: int
    decomp: int
    shape: tuple
    p1: int = 1
    p2: int = 1
    transform: int = dfft.C2C
    kinds: tuple | None = None
    prec: int = dfft.F64
    comm: int = 0
    send: int = 0
    batch: int | None = None
    inplace: bool = False
    spectral: tuple | None = None
    components: int | None = None
    axes: tuple | None = None
    scale: tuple | None = None
    in_boxes: tuple | None = None
    out_boxes: tuple | None = None
    embed: str | None = None
    halo: int = 2
    gap: int = 0
    data: tuple | None = None

    @property
    def fields(self):
        return 1 if self.batch is None else self.batch


def _flat(boxes):
    return None if boxes is None else (C.c_size_t * (6 * len(boxes)))(*[v for lo, hi in boxes for v in (*lo, *hi)])


def strides(size, halo, gap):
    """{field, x, y} of a block of `size` inside its ghost layers"""
    y = size[2] + 2 * halo
    x = (size[1] + 2 * halo) * y
    return (size[0] + 2 * halo) * x + gap, x, y


def create(p, rank, comm=None):
    """rank's plan of p on comm (a geometry-only communicator when None) with its strides, before the other setters:
    (rc, message, comm, plan)"""
    c = comm
    if c is None:
        c = C.c_void_p()
        check(lib().dfft_comm_create_dry(rank, p.P, C.byref(c)))
    cfg = C.byref(_lib.dfft_config(1, 0, p.comm, p.send, None, p.comm, p.send))
    plan = C.c_void_p()
    head = (c, cfg, p.decomp, p.prec)
    if p.data is not None:
        assert p.in_boxes is None and p.out_boxes is None and p.embed is None and p.components is None and p.kinds is None and not p.inplace
        k = None if p.spectral is None else (C.c_size_t * 3)(*p.spectral)
        rc = lib().dfft_plan_create_pruned(*head, p.transform, *p.shape, (C.c_size_t * 3)(*p.data), k, p.p1, p.p2, p.fields, 1, C.byref(plan))
    elif p.in_boxes is not None or p.out_boxes is not None:
        rc = lib().dfft_plan_create_boxes(*head, p.transform, *p.shape, p.p1, p.p2, _flat(p.in_boxes), _flat(p.out_boxes), p.fields, 1,
                                          C.byref(plan))
    elif p.spectral is not None:
        rc = lib().dfft_plan_create_padded(*head, p.transform, *p.shape, *p.spectral, p.p1, p.p2, p.fields, 1, C.byref(plan))
    elif p.components is not None:
        rc = lib().dfft_plan_create_interleaved(*head, p.transform, *p.shape, p.p1, p.p2, p.components, p.fields, 1, C.byref(plan))
    elif p.kinds is not None:
        rc = lib().dfft_plan_create_r2r(*head, (C.c_int * 3)(*p.kinds), *p.shape, p.p1, p.p2, p.fields, int(p.inplace), 1, C.byref(plan))
    elif p.inplace:
        rc = lib().dfft_plan_create_inplace(*head, p.transform, *p.shape, p.p1, p.p2, p.fields, 1, C.byref(plan))
    elif p.batch is not None:
        rc = lib().dfft_plan_create_batched(*head, p.transform, *p.shape, p.p1, p.p2, p.batch, 1, C.byref(plan))
    else:
        rc = lib().dfft_plan_create(*head, p.transform, *p.shape, p.p1, p.p2, 1, C.byref(plan))
    if rc == 0 and p.embed:
        sides = []
        for fn, name in ((lib().dfft_get_in_size, "in"), (lib().dfft_get_out_size, "out")):
            s = (C.c_size_t * 3)()
            check(fn(plan, s))
            sides.append((C.c_longlong * 3)(*strides(list(s), p.halo, p.gap)) if p.embed in (name, "both") else None)
        rc = lib().dfft_plan_set_strides(plan, *sides)
    return rc, (lib().dfft_last_error_string() or b"").decode(), c, plan


def layouts(plan):
    """[(size, start)] of layouts 0..3 of this rank"""
    out = []
    for w in range(4):
        s, o = (C.c_size_t * 3)(), (C.c_size_t * 3)()
        if w == 0:
            check(lib().dfft_get_in_size(plan, s)); check(lib().dfft_get_in_start(plan, o))
        else:
            check(lib().dfft_get_partial_size(plan, w, s)); check(lib().dfft_get_partial_start(plan, w, o))
        out.append(([int(v) for v in s], [int(v) for v in o]))
    return out


def describe_raw(plan, inverse, d):
    need = C.c_size_t()
    check(lib().dfft_plan_describe(plan, inverse, d, None, 0, C.byref(need)))
    buf = C.create_string_buffer(need.value)
    check(lib().dfft_plan_describe(plan, inverse, d, buf, need.value, C.byref(need)))
    return buf.value.decode()


def set_options(p, plan):
    """the setters that follow the creator: transform axes and scale"""
    if p.axes is not None:
        check(lib().dfft_plan_set_transform_axes(plan, (C.c_int * 3)(*p.axes)))
    if p.scale is not None:
        check(lib().dfft_plan_set_scale(plan, *p.scale))


@contextmanager
def dry_plans(p, ranks=None):
    """the dry plans of p's ranks (all of them when None) with every setter applied: a list of plan handles, destroyed on
    exit"""
    made = []
    try:
        for r in range(p.P) if ranks is None else ranks:
            rc, msg, c, plan = create(p, r)
            made.append((c, plan))
            assert rc == 0, msg
            set_options(p, plan)
        yield [plan for _, plan in made]
    finally:
        for c, plan in made:
            lib().dfft_plan_destroy(plan)
            lib().dfft_comm_destroy(c)


def schedule(p, plan, inverse, d):
    """the parsed step list of an open plan, with "domain_bytes", "work_bytes" and "layouts" ([(size, start)] of layouts
    0..3)"""
    assert lib().dfft_get_batch(plan) == p.fields and lib().dfft_get_components(plan) == (p.components or 1)
    sc = json.loads(describe_raw(plan, inverse, d))
    sc["domain_bytes"] = lib().dfft_get_domain_size(plan)
    sc["work_bytes"] = lib().dfft_get_work_size_device(plan)
    sc["layouts"] = layouts(plan)
    return sc


def describe_text(p, rank, inverse, d):
    """rank's step list as dfft_plan_describe writes it"""
    with dry_plans(p, [rank]) as (plan,):
        return describe_raw(plan, inverse, d)


def describe(p, rank, inverse, d):
    """rank's parsed step list (see schedule)"""
    with dry_plans(p, [rank]) as (plan,):
        return schedule(p, plan, inverse, d)


# ---- per-pass math --------------------------------------------------------------------------------------------------------
def positions(n, k, half=False):
    """line positions of the k kept spectral indices of an n-point axis (half: the R2C z axis, k modes kept of n/2+1)"""
    if half:
        return np.arange(k // 2 + 1)
    return np.fft.fftfreq(k, 1.0 / k).astype(np.int64) % n


def r2hc(x, axis):
    """hc = [Re X_0 .. Re X_{N/2}, Im X_{N/2-1} .. Im X_1] along axis, X = rfft(x)"""
    n = x.shape[axis]
    X = np.fft.rfft(x, axis=axis)
    return np.concatenate([X.real, np.take(X.imag, np.arange(n // 2 - 1, 0, -1), axis=axis)], axis=axis)


def hc2r(h, axis):
    """the unnormalised inverse: hc2r(r2hc(x)) = N x"""
    n = h.shape[axis]
    re = np.take(h, np.arange(n // 2 + 1), axis=axis)
    im = np.zeros_like(re)
    idx = [slice(None)] * h.ndim
    idx[axis] = slice(1, n // 2)
    im[tuple(idx)] = np.take(h, np.arange(n - 1, n // 2, -1), axis=axis)
    return np.fft.irfft(re + 1j * im, n=n, axis=axis) * n


R2R = {  # the real-to-real pass (kinds 4 / 5) on lines along axis 2, by the name its description gives
    "dct": lambda x, inv: sf.dct(x, type=3 if inv else 2, axis=2),
    "dst": lambda x, inv: sf.dst(x, type=3 if inv else 2, axis=2),
    "r2hc": lambda x, inv: hc2r(x, 2) if inv else r2hc(x, 2),
    "dct1": lambda x, inv: sf.dct(x, type=1, axis=2),  # its own inverse up to 2N: both directions run it
    "dst1": lambda x, inv: sf.dst(x, type=1, axis=2),
}


def _c2c(st, x, N):
    return np.fft.ifft(x, axis=2) * N if st["inverse"] else np.fft.fft(x, axis=2)


def _r2c_pairs(st, x, N):
    """R2C: N complex units = 2N reals in, N + 1 complex out"""
    return np.fft.rfft(np.ascontiguousarray(x[..., 0]).view(np.float64), axis=2)[..., None]


def _c2r_pairs(st, x, N):
    return np.ascontiguousarray(np.fft.irfft(x[..., 0], n=2 * N, axis=2) * (2 * N)).view(np.complex128)[..., None]


# kind: (N -> (points in, points out), real view in, real view out, math on data[a0, a1, n, b]; None: the R2R pass)
PASSES = {
    0: (lambda N: (N, N), False, False, _c2c),
    1: (lambda N: (N, N), False, False, _c2c),
    2: (lambda N: (N, N + 1), False, False, _r2c_pairs),
    3: (lambda N: (N + 1, N), False, False, _c2r_pairs),
    4: (lambda N: (N, N), False, False, None),
    5: (lambda N: (N, N), False, False, None),
    6: (lambda N: (N, N), False, False, lambda st, x, N: x),  # copies of a kept axis
    7: (lambda N: (N, N), False, False, lambda st, x, N: x),
    8: (lambda N: (N, N), False, False, _c2c),  # interleaved components: b is the component
    9: (lambda N: (N, N // 2 + 1), True, False, lambda st, x, N: np.fft.rfft(x, axis=2)),  # real side counted in reals
    10: (lambda N: (N // 2 + 1, N), False, True, lambda st, x, N: np.fft.irfft(x, n=N, axis=2) * N),
}


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


# ---- memory, views and the happens-before check -------------------------------------------------------------------------
class Memory:
    """arrays keyed by synthetic base address; es = bytes per element of the plan (complex, or real for R2R plans): the
    replay computes in double, only the address arithmetic follows the plan's precision"""

    def __init__(self, es, dtype=np.complex128):
        self.regions = []  # (base_bytes, array)
        self.es, self.dtype = es, dtype

    def add(self, base, nelem):
        arr = np.zeros(nelem, dtype=self.dtype)
        self.regions.append((base, arr))
        return arr

    def resolve(self, addr):
        for base, arr in self.regions:
            if base <= addr < base + arr.size * self.es:
                assert (addr - base) % self.es == 0
                return arr, (addr - base) // self.es
        raise KeyError(hex(addr))


class Ordering:
    """Happens-before check of a set of per-rank step lists (what the lock-step replay cannot see: a step that runs on
    another plan stream than its producer is only ordered behind it through an event, and a step that reads what a peer
    stored only through a rendezvous).  Per rank: step k's ancestors = the previous step on its stream + the steps that
    recorded the events it waits for (the auxiliary streams fork from the caller's stream before step 0).  Across ranks:
    everything before rank a's j-th rendezvous of a group happens before everything after rank b's j-th rendezvous of
    that group.  Every read-after-write and write-after-read on memory must be covered by one of the two."""

    def __init__(self, scheds):
        self.scheds = scheds
        self.anc, self.rdv = [], []  # per rank: ancestor bit masks; {(phase_id): [step indices]}
        for sc in scheds:
            anc, last, recorded, rdv = [], {}, {}, {}
            for k, st in enumerate(sc["steps"]):
                preds = [last[st["stream"]]] if st["stream"] in last else []
                for w in st["waits"]:
                    assert w in recorded, f"rank {sc['rank']} step {k} ({st['label']}) waits for event {w} that no earlier step records"
                    preds.append(recorded[w])
                m = 0
                for q in preds:
                    m |= anc[q] | (1 << q)
                anc.append(m)
                if st["record"] >= 0:
                    recorded[st["record"]] = k
                last[st["stream"]] = k
                if st["type"] == 1:
                    rdv.setdefault(st["phase_id"], []).append(k)
            self.anc.append(anc)
            self.rdv.append(rdv)
        self.last_w, self.last_r = {}, {}

    def before(self, a, ka, b, kb):
        """step ka of rank a happens before step kb of rank b"""
        if a == b:
            return ka == kb or bool(self.anc[a][kb] >> ka & 1)
        for g, mine in self.rdv[a].items():
            theirs = self.rdv[b].get(g, [])
            if b not in self.scheds[a]["steps"][mine[0]]["members"]:
                continue
            for ra, rb in zip(mine, theirs):
                if (ra == ka or self.anc[a][ra] >> ka & 1) and (rb == kb or self.anc[b][kb] >> rb & 1):
                    return True
        return False

    def _tables(self, key, size):
        if key not in self.last_w:
            self.last_w[key] = np.full((2, size), -1, dtype=np.int64)
            self.last_r[key] = np.full((2, size), -1, dtype=np.int64)
        return self.last_w[key], self.last_r[key]

    @staticmethod
    def _steps(table, idx, skip):
        """the distinct (rank, step) pairs of table at idx, without (-1, -1) and skip"""
        u = np.unique(table[0, idx] << 32 | table[1, idx])
        return {(int(v >> 32), int(v & 0xFFFFFFFF)) for v in u[u >= 0]} - {skip}

    def read(self, r, k, key, size, idx):
        lw, lr = self._tables(key, size)
        idx = np.asarray(idx).ravel()
        for q, kq in self._steps(lw, idx, None):
            assert self.before(q, kq, r, k), (f"rank {r} step {k} ({self.scheds[r]['steps'][k]['label']}) reads what rank {q} step {kq} "
                                              f"({self.scheds[q]['steps'][kq]['label']}) wrote, without an event / rendezvous path between them")
        lr[0, idx], lr[1, idx] = r, k

    def write(self, r, k, key, size, idx):
        lw, lr = self._tables(key, size)
        idx = np.asarray(idx).ravel()
        for q, kq in self._steps(lr, idx, (r, k)):
            assert self.before(q, kq, r, k), (f"rank {r} step {k} ({self.scheds[r]['steps'][k]['label']}) overwrites what rank {q} step {kq} "
                                              f"({self.scheds[q]['steps'][kq]['label']}) reads, without an event / rendezvous path between them")
        for q, kq in self._steps(lw, idx, (r, k)):
            assert self.before(q, kq, r, k), f"rank {r} step {k} overwrites rank {q} step {kq}'s output without ordering"
        lw[0, idx], lw[1, idx] = r, k


def view_indices(view, A0, A1, N, B, user_base=None):
    """flat (array, index) for every element (a0, a1, n, b) of a view, as index arrays per segment"""
    out = []
    seg_of_n = np.array(view["seg_of_n"], dtype=np.int64) if view["nseg"] > 1 else np.zeros(N, dtype=np.int64)
    a0 = np.arange(A0)[:, None, None, None]
    a1 = np.arange(A1)[None, :, None, None]
    b = np.arange(B)[None, None, None, :]
    for s, seg in enumerate(view["segs"]):
        ns = np.nonzero(seg_of_n[:N] == s)[0]
        if ns.size == 0:
            continue
        n = ns[None, None, :, None]
        off = a0 * seg["sA0"] + a1 * seg["sA1"] + (n - seg["n0"]) * view["sN"] + b
        base = seg["base"] if user_base is None else user_base + seg["base"]
        out.append((base, ns, off))
    return out


def _owners(acc):
    """acc: [(array, flat indices, group ids broadcastable to them)]: per array, (sorted distinct indices, the one group that
    touches each, or -2 where several do)"""
    by = {}
    for arr, idx, grp in acc:
        by.setdefault(id(arr), []).append((np.ravel(idx), np.broadcast_to(grp, np.shape(idx)).ravel()))
    out = {}
    for key, parts in by.items():
        i = np.concatenate([p[0] for p in parts])
        g = np.concatenate([p[1] for p in parts])
        if i.size == 0:
            continue
        o = np.argsort(i, kind="stable")
        i, g = i[o], g[o]
        start = np.flatnonzero(np.r_[True, i[1:] != i[:-1]])
        lo, hi = np.minimum.reduceat(g, start), np.maximum.reduceat(g, start)
        out[key] = (i[start], np.where(lo == hi, lo, -2))
    return out


def _line_check(r, k, st, reads, writes):
    """reads / writes: [(array, flat indices, line ids)] of one step: a line writes only what it reads itself or what no
    other line of the step reads"""
    table = _owners(reads)
    for arr, idx, line in writes:
        if id(arr) not in table:
            continue
        u, rl = table[id(arr)]
        i, l = np.ravel(idx), np.broadcast_to(line, np.shape(idx)).ravel()
        pos = np.minimum(np.searchsorted(u, i), u.size - 1)
        reader = np.where(u[pos] == i, rl[pos], -1)
        bad = (reader != -1) & (reader != l)
        assert not bad.any(), (f"rank {r} step {k} ({st['label']}): line {int(l[bad][0])} writes an element that line {int(reader[bad][0])} "
                               f"reads (or that several lines read)")


def _phase_check(r, k, acc):
    """the two phases of a two-phase kernel (steps k-1 and k): every element is touched by one plane / field only"""
    for u, g in _owners(acc).values():
        assert (g >= 0).all(), f"rank {r} steps {k - 1}/{k}: the two phases of one launch share elements across planes / fields"


# ---- the caller's buffers -------------------------------------------------------------------------------------------------
class Side:
    """one rank's caller buffer on one side (in / out) of an exec: where field f's block of layout `which` lies.  On a side
    with strides (in_strides / out_strides of the describe, in the side's elements: reals on the real side of R2C / C2R)
    the block lies inside ghost layers: field f's block starts `lead` elements into the buffer, behind those of field 0."""

    def __init__(self, p, sc, which, pairs, es):
        self.size, self.start = sc["layouts"][which]
        comps = p.components or 1
        self.shape = tuple(self.size) + ((comps,) if p.components else ())
        self.pairs = pairs  # the real side of an R2C / C2R plan, stored as complex pairs like the kernels read it
        self.nz = self.size[2]
        self.padded = pairs and p.inplace  # in place: real rows padded to Nz/2 + 1 complex units
        self.row = self.nz // 2 + 1 if self.padded else self.nz * comps // (2 if pairs else 1)
        self.elems = self.size[0] * self.size[1] * self.row
        self.field = sc["domain_bytes"] // es if p.inplace else self.elems
        self.sx, self.sy, self.lead = self.size[1] * self.row, self.row, 0
        st = sc.get("in_strides") if which == 0 else sc.get("out_strides") if which == 3 else None
        self.strided = st is not None
        if self.strided:
            unit = 2 if pairs else 1  # the buffer counts pairs of reals on the real side of R2C / C2R
            assert all(v % unit == 0 for v in st) and p.halo * (st[1] + st[2] + 1) % unit == 0, (st, p.halo)
            self.field, self.sx, self.sy = (v // unit for v in st)
            self.lead = p.halo * (st[1] + st[2] + 1) // unit
        self.total = max(p.fields * self.field, 1)  # elements of the buffer

    def rows(self, f):
        n0, n1, _ = self.size
        i = (np.arange(n0)[:, None] * self.sx + np.arange(n1)[None, :] * self.sy).reshape(-1, 1) + np.arange(self.row)
        return self.lead + f * self.field + i

    def index(self, f):
        """flat buffer indices of field f's block (the padding of real rows excluded)"""
        i = self.rows(f)
        return (i[:, :self.nz // 2] if self.padded else i).ravel()

    def put(self, buf, f, block):
        v = np.ascontiguousarray(block, dtype=buf.real.dtype if self.pairs else buf.dtype).ravel()
        buf[self.index(f)] = v.view(buf.dtype)

    def get(self, buf, f):
        v = buf[self.index(f)]
        return (v.view(v.real.dtype) if self.pairs else v).reshape(self.shape)


def sides(p, sc, inverse, d, es):
    """(input side, output side) of the rank whose step list is sc"""
    r2c = p.transform == dfft.R2C and p.kinds is None
    src_w, dst_w = (d, 0) if inverse else (0, d)
    return Side(p, sc, src_w, r2c and not inverse, es), Side(p, sc, dst_w, r2c and bool(inverse), es)


def block(a, start, size):
    return a[start[0]:start[0] + size[0], start[1]:start[1] + size[1], start[2]:start[2] + size[2]]


def assemble(outs):
    """the global output (field, ...) from [field][rank] (start of the output block, output block)"""
    blocks = outs[0]
    shape = tuple(max(s[a] + b.shape[a] for s, b in blocks) for a in range(3)) + blocks[0][1].shape[3:]
    g = np.zeros((len(outs),) + shape, dtype=blocks[0][1].dtype)
    for f, blocks in enumerate(outs):
        for s, b in blocks:
            block(g[f], s, b.shape)[...] = b
    return g


# ---- the engine -----------------------------------------------------------------------------------------------------------
def replay(p, inverse, d, x, scheds=None, mutate=None):
    """Runs the step lists of every rank of plan p (scheds: as describe returns them, built here when None; mutate: a hook
    that breaks them on purpose, for negative tests) in lock step on x, the global input of the direction: [field][x, y, z]
    (+ [c] for interleaved plans), real on the real side of R2C plans and for R2R plans.  Returns [field][rank] (start of the
    output block, output block)."""
    if scheds is None:
        with dry_plans(p) as plans:
            scheds = [schedule(p, plan, inverse, d) for plan in plans]
    if mutate:
        mutate(scheds)
    return _Replay(p, scheds, inverse, d).run(x)


def error(outs, want):
    """worst rel-L2 error of the output blocks of replay against the same blocks of want[field]"""
    worst = 0.0
    for f, blocks in enumerate(outs):
        for (s0, s1, s2), got in blocks:
            worst = max(worst, O.rel_l2(got, want[f][s0:s0 + got.shape[0], s1:s1 + got.shape[1], s2:s2 + got.shape[2]]))
    return worst


class _Replay:
    def __init__(self, p, scheds, inverse, d):
        self.p, self.scheds, self.inverse, self.d = p, scheds, inverse, d
        sc0 = scheds[0]
        self.real = "r2r" in sc0  # R2R plans: real elements everywhere
        self.es = es = sc0["esize"]
        assert es == {dfft.F64: 16, dfft.F32: 8, dfft.F16: 4, dfft.BF16: 4}[p.prec] // (2 if self.real else 1), es
        self.r2c = p.transform == dfft.R2C and not self.real
        self.mem = Memory(es, np.float64 if self.real else np.complex128)
        self.owner = {}  # id(slot array) -> (rank, slot)
        for r, sc in enumerate(scheds):
            assert sc.get("inplace", False) == p.inplace
            for s in range(sc["nslots"]):
                self.owner[id(self.mem.add(sc["slots"][s][r], sc["slot_bytes"] // es))] = (r, s)
        self.poison = POISON.real if self.real else POISON
        self.sides, self.bufs, self.pads, self.masks = [], [], [], []
        for r, sc in enumerate(scheds):
            i, o = sides(p, sc, inverse, d, es)
            if "field_in" in sc:
                assert (sc["field_in"], sc["field_out"]) == (i.field * es, o.field * es), (sc["field_in"], sc["field_out"], i.field, o.field)
            if p.inplace:
                assert i.field >= max(i.elems, o.elems) and o.field == i.field
                one = self.mem.add(USER_IN + (r << 48), i.total)
                bufs = {1: one, 2: one}
            else:  # a buffer with strides starts `lead` elements before the address the passes take
                bufs = {1: self.mem.add(USER_IN + (r << 48) - i.lead * es, i.total),
                        2: self.mem.add(USER_OUT + (r << 48) - o.lead * es, o.total)}
            masks = {}  # caller buffers with strides: True on the blocks, poison on every ghost element
            for user, side in ((1, i), (2, o)):
                if side.strided:
                    masks[user] = np.zeros(bufs[user].size, dtype=bool)
                    for f in range(p.fields):
                        masks[user][side.index(f)] = True
                    bufs[user][~masks[user]] = self.poison
            self.masks.append(masks)
            pad = None
            if i.padded or o.padded:  # in place: the real rows' padding, never read (forward) or stored by C2R (inverse)
                pad = np.zeros(bufs[1].size, dtype=bool)
                side = i if i.padded else o
                for f in range(p.fields):
                    pad[side.rows(f)[:, side.nz // 2:].ravel()] = True
            self.sides.append({1: i, 2: o})
            self.bufs.append(bufs)
            self.pads.append(pad)
        self.scaled = any("scale" in st for sc in scheds for st in sc["steps"])
        self.counts = {}  # output array -> how often each (real) element was scaled

    # -- steps -----------------------------------------------------------------------------------------------------------
    def run(self, x):
        p, P, scheds = self.p, self.p.P, self.scheds
        for r in range(P):
            i = self.sides[r][1]
            for f in range(p.fields):
                (s0, s1, s2), (n0, n1, n2) = i.start, i.size
                i.put(self.bufs[r][1], f, x[f][s0:s0 + n0, s1:s1 + n1, s2:s2 + n2])
            if self.pads[r] is not None and not self.inverse:
                self.bufs[r][1][self.pads[r]] = PAD
        inputs = [self.bufs[r][1].copy() for r in range(P)]
        nsteps = len(scheds[0]["steps"])
        assert all(len(sc["steps"]) == nsteps for sc in scheds), [len(sc["steps"]) for sc in scheds]
        self.order = Ordering(scheds)
        self.last_remote_write, self.last_rdv, self.prev_acc, self.holes, self.data_holes = {}, [-1] * P, {}, 0, 0
        for k in range(nsteps):
            pending = []  # stores of step k land after every rank's loads of step k
            for r in range(P):
                st = scheds[r]["steps"][k]
                if st["type"] == 1:
                    self.last_rdv[r] = k
                elif st["type"] == 2:
                    self.exchange(r, k, st, pending)
                else:
                    self.run_pass(r, k, st, pending)
            for arr, tgt, idx, cidx, val, who in pending:
                self.order.write(who, k, id(arr), arr.size, cidx)
                tgt[idx] = val
        if p.spectral is not None and any(p.spectral[a] != p.shape[a] for a in (2, 1, 0)[:self.d]):
            assert self.holes > 0, "a padded plan that truncates one of its first d axes runs no hole pass"
        if p.data is not None and any(p.data[a] != p.shape[a] for a in (2, 1, 0)[:self.d]):
            assert self.data_holes > 0, "a pruned plan with data smaller than one of its first d axes runs no pass with a data hole"
        outs = [[] for _ in range(p.fields)]
        for r in range(P):
            if not p.inplace:
                assert np.array_equal(self.bufs[r][1], inputs[r]), f"rank {r}: the input was modified"
            if self.pads[r] is not None and not self.inverse:
                assert (self.bufs[r][1][self.pads[r]] == PAD).all(), f"rank {r}: the padding of a real row was stored into"
            for user, mask in self.masks[r].items():
                assert (self.bufs[r][user][~mask] == self.poison).all(), f"rank {r}: a ghost element of caller buffer {user} changed"
            o = self.sides[r][2]
            for f in range(p.fields):
                outs[f].append((o.start, o.get(self.bufs[r][2], f)))
                if self.scaled:
                    cnt = self.counts.get(id(self.bufs[r][2]), np.zeros(0, dtype=np.int64))
                    cnt = cnt.reshape(-1, 1 if self.real else 2)[o.index(f)] if cnt.size else np.zeros(o.index(f).size, dtype=np.int64)
                    assert (cnt == 1).all(), f"rank {r} field {f}: an output value is scaled {int(cnt.min())}..{int(cnt.max())} times"
        return outs

    def exchange(self, r, k, st, pending):
        """all-to-all-v between staging slots: what r sends lands in q's stream order (ncclRecv)"""
        scheds, es = self.scheds, self.es
        sb = scheds[r]["slots"][st["send_slot"]][r]
        for peer in st["peers"]:
            q = peer["rank"]
            mine = [pp for pp in scheds[q]["steps"][k]["peers"] if pp["rank"] == r][0]
            assert mine["rcount"] == peer["scount"], f"step {k}: rank {r} sends {peer['scount']} to rank {q}, which receives {mine['rcount']}"
            n = peer["scount"]
            src, so = self.mem.resolve(sb + peer["soff"] * es)
            dst, do = self.mem.resolve(scheds[q]["slots"][st["recv_slot"]][q] + mine["roff"] * es)
            self.order.read(r, k, id(src), src.size, np.arange(so, so + n))
            idx = np.arange(do, do + n)
            pending.append((dst, dst, idx, idx, src[so:so + n].copy(), q))

    def access(self, r, k, st, which, n, b, real):
        """[(array, indexed array, index, index in array elements, ns)] per segment of view `which` of pass st; a real view
        (the real side of kinds 9 / 10) indexes the float64 view of its complex array"""
        user = st[which + "_user"]
        ub = {1: USER_IN, 2: USER_IN if self.p.inplace else USER_OUT}[user] + (r << 48) if user else None
        mask = self.masks[r].get(user) if user else None
        out = []
        for base, ns, off in view_indices(st[which], st["A0"], st["A1"], n, b, ub):
            if off.size == 0:  # empty tail passes of ranks without leftover columns
                continue
            arr, o = self.mem.resolve(base)
            tgt, idx = (arr.view(np.float64), 2 * o + off) if real else (arr, o + off)
            cidx = idx // 2 if real else idx
            if mask is not None:
                bad = ~mask[cidx]
                assert not bad.any(), (f"rank {r} step {k} ({st['label']}) {'reads' if which == 'in' else 'stores into'} "
                                       f"{int(bad.sum())} ghost elements of caller buffer {user}")
            if not user:
                own = self.owner.get(id(arr))
                assert own is not None, f"rank {r} step {k} ({st['label']}): a slot view outside the slots"
                if which == "in":  # the gathers of box plans' output reshape read their peers' slots
                    assert own[0] == r or st["label"] == "reshape out", "passes other than the output gathers read only local memory"
                    w = self.last_remote_write.get(own, -1)
                    assert w < 0 or w < self.last_rdv[r] <= k, f"rank {r} step {k} reads slot {own} written remotely at step {w} without a rendezvous"
                elif own[0] != r:
                    assert self.last_rdv[r] >= 0, f"rank {r} writes into rank {own[0]}'s slot before its entry rendezvous"
                    self.last_remote_write[own] = k
            out.append((arr, tgt, idx, cidx, ns))
        return out

    def check_bounds(self, r, k, st, which, acc):
        """every access lies inside its array, and a per-field step inside its field of the caller's buffers"""
        user, field = st[which + "_user"], st.get("field", -1)
        for arr, _, _, cidx, _ in acc:
            lo, hi = int(cidx.min()), int(cidx.max())
            assert 0 <= lo and hi < arr.size, f"rank {r} step {k} ({st['label']}) leaves its array: [{lo}, {hi}] of {arr.size}"
            if user and field >= 0:
                per = self.sides[r][user].field
                assert field * per <= lo and hi < (field + 1) * per, (f"rank {r} step {k} ({st['label']}) touches caller buffer {user} at "
                                                                      f"[{lo}, {hi}] outside field {field}")

    def check_kind(self, r, k, st, N):
        kind, p = st["kind"], self.p
        where = f"rank {r} step {k} ({st['label']}, kind {kind})"
        if kind == 6 and st["label"].startswith("reshape"):  # box plans: the copies between the boxes and the natural layouts
            assert p.in_boxes is not None or p.out_boxes is not None, where
            assert "n" in st and st["log2n"] == 0 and "r2r" not in st and st["B"] == 1, where
            return
        assert kind in PASSES, f"{where}: unknown pass kind"
        assert (kind in (4, 5, 6, 7)) if self.real else (kind not in (4, 5)), where
        if kind in (0, 1, 8) and "n" in st:  # Bluestein: log2n = log2 M, M >= 2n - 1 > M / 2
            M = 1 << st["log2n"]
            assert N & (N - 1) and 2 * N - 1 <= M < 4 * N - 2, where
        if kind in (2, 3):
            assert st["B"] == 1, where
        if kind in (4, 5):
            assert st.get("r2r", self.scheds[r].get("r2r")) in R2R, where
            if "n" in st:
                assert st["r2r"] in ("dct1", "dst1") and N == (1 << st["log2n"]) + (1 if st["r2r"] == "dct1" else -1), where
        if kind in (6, 7):  # copies move the kept axes of plans that have them
            assert p.axes is not None and not all(p.axes), where
            assert "n" in st and st["log2n"] == 0 and "r2r" not in st, where
            assert st["label"].split()[0] in "xyz" and "copy" in st["label"], where
        if kind in (8, 9, 10):
            assert st["B"] == p.components and st["in"]["sN"] == p.components and st["out"]["sN"] == p.components, where
        if (p.components or 1) > 1:
            assert kind in ((1, 9, 10) if self.r2c else (1, 8)), where
        if "keep" in st:
            self.holes += 1
            assert kind in (0, 1, 2, 3) and 1 <= st["keep"] < (N + 1 if kind in (2, 3) else N), where
        if "data" in st:
            self.data_holes += 1
            assert kind in (0, 1, 2, 3) and 1 <= st["data"] < (2 * N if kind in (2, 3) else N), where
            assert kind not in (2, 3) or st["data"] % 2 == 0, where

    def run_pass(self, r, k, st, pending):
        kind = st["kind"]
        N = st.get("n", 1 << st["log2n"])
        self.check_kind(r, k, st, N)
        points, real_in, real_out, math = PASSES[kind]
        n_in, n_out = points(N)
        b = 1 if kind in (2, 3) else st["B"]
        A0, A1 = st["A0"], st["A1"]
        # the line positions a side holds (None: all), the rest of the line being zero: padded plans keep the "keep"
        # spectral indices (out forward, in inverse), pruned plans the positions [0, "data") of the physical side (in
        # forward, out inverse; R2C / C2R: data reals, data / 2 pairs).  The pairs and the R2C half spectrum are prefixes.
        pairs = kind in (2, 3)
        spec = None if "keep" not in st else np.arange(st["keep"]) if pairs else positions(N, st["keep"])
        phys = None if "data" not in st else np.arange(st["data"] // 2 if pairs else st["data"])
        at_in, at_out = (spec, phys) if st["inverse"] else (phys, spec)
        kin = n_in if at_in is None else at_in.size
        kout = n_out if at_out is None else at_out.size
        reads = self.access(r, k, st, "in", kin, b, real_in)
        writes = self.access(r, k, st, "out", kout, b, real_out)
        data = np.zeros((A0, A1, kin, b), dtype=np.float64 if self.real or real_in else np.complex128)
        for arr, tgt, idx, cidx, ns in reads:
            data[:, :, ns, :] = tgt[idx]
            self.order.read(r, k, id(arr), arr.size, cidx)
        self.check_buffer(r, k, st, reads, writes)
        self.check_bounds(r, k, st, "in", reads)
        self.check_bounds(r, k, st, "out", writes)
        if at_in is not None:
            full = np.zeros((A0, A1, n_in, b), dtype=data.dtype)
            full[:, :, at_in, :] = data
            data = full
        if math is None:
            res = R2R[st.get("r2r", self.scheds[r].get("r2r"))](data, st["inverse"])
        else:
            res = math(st, data, N)
        if at_out is not None:
            res = res[:, :, at_out, :]
        if "scale" in st:
            res = res * st["scale"]
            for arr, tgt, idx, cidx, ns in writes:
                assert st["out_user"] == 2, f"rank {r} step {k} ({st['label']}): only stores into the caller's output are scaled"
                units = 1 if self.real else 2  # count real elements: a complex unit is two
                cnt = self.counts.setdefault(id(arr), np.zeros(arr.size * units, dtype=np.int64))
                if tgt is arr:
                    for j in range(units):
                        np.add.at(cnt, units * idx.ravel() + j, 1)
                else:
                    np.add.at(cnt, idx.ravel(), 1)
        if self.p.prec in (dfft.F16, dfft.BF16):
            res = store16(st, res, self.p.prec)
        for arr, tgt, idx, cidx, ns in writes:
            pending.append((arr, tgt, idx, cidx, res[:, :, ns, :], r))

    def check_buffer(self, r, k, st, reads, writes):
        """the line check, the padding rules of in-place R2C / C2R plans and the phases of two-phase stages"""
        A0, A1, b = st["A0"], st["A1"], 1 if st["kind"] in (2, 3) else st["B"]
        line = (np.arange(A0)[:, None, None, None] * A1 + np.arange(A1)[None, :, None, None]) * b + np.arange(b)[None, None, None, :]
        read_arrays = {id(a[0]) for a in reads}
        if any(id(w[0]) in read_arrays for w in writes):
            _line_check(r, k, st, [(a, c, line) for a, _, _, c, _ in reads], [(a, c, line) for a, _, _, c, _ in writes])
        pad = self.pads[r]
        if pad is not None:
            buf = self.bufs[r][1]
            for is_read, acc in ((True, reads), (False, writes)):
                for arr, _, _, cidx, _ in acc:
                    if arr is not buf:
                        continue
                    # forward: the padding of the real input rows is not read (until a complex pass has stored there);
                    # inverse: the C2R pass does not store into it
                    if (is_read and not self.inverse) or (not is_read and st["kind"] == 3):
                        assert not pad[cidx].any(), f"rank {r} step {k} ({st['label']}) touches the padding of a real row"
                    elif not self.inverse:
                        pad[cidx] = False
        # the fused z + y stage and the batched stage: both listed phases run concurrently (planes / fields apart)
        if st["label"].startswith(("zy pass", "yz pass", "batched pass")):
            batched = st["label"].startswith("batched")
            groups = self.p.fields if batched else self.p.shape[0]
            grp = np.arange(A0)[:, None, None, None] * groups // A0
            acc = [(a, c, grp) for a, _, _, c, _ in reads + writes]
            if self.prev_acc.get(r) is not None:
                _phase_check(r, k, self.prev_acc[r] + acc)
                self.prev_acc[r] = acc if batched else None
            else:
                self.prev_acc[r] = acc
        else:
            self.prev_acc[r] = None
