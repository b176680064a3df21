"""Host-side mirror of the reference's plan classes over the C ABI (include/dfft.h).

Class and method names follow /root/reference/include/mpicufft.hpp:55-105,
mpicufft_slab.hpp:88-125, mpicufft_slab_z_then_yx.hpp and mpicufft_pencil.hpp:71-122, so caller code
written against the reference reads the same; MPI_Comm becomes `Comm`.
Buffers are CUDA device memory: torch tensors (their .data_ptr() is used) or raw integer addresses.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional, Sequence

from . import _lib
from ._lib import check, lib
from .params import CommunicationMethod, Configurations, GlobalSize, Partition, SendMethod

SLAB_ZY_THEN_X, SLAB_Z_THEN_YX, PENCIL = 0, 1, 2
F32, F64, F16, BF16 = 0, 1, 2, 3
R2C, C2C, DCT, DST, R2HC = 0, 1, 2, 3, 4
DCT1, DST1 = 16, 17  # type-I kinds (DCT-I / DST-I): per-axis plans and fft1d_r2r only
DCT4, DST4 = 19, 20  # type-IV kinds (DCT-IV / DST-IV): per-axis plans and fft1d_r2r only
_R2R_KINDS = {"dct": DCT, "dst": DST, "r2hc": R2HC, "dct1": DCT1, "dst1": DST1, "dct4": DCT4, "dst4": DST4}
FORWARD, INVERSE = -1, 1


def _ptr(buf) -> int:
    if buf is None:
        return 0
    if isinstance(buf, int):
        return buf
    if hasattr(buf, "data_ptr"):
        if hasattr(buf, "is_contiguous") and not buf.is_contiguous():
            raise ValueError("buffers must be contiguous ([x][y][z], z fastest)")
        if hasattr(buf, "is_cuda") and not buf.is_cuda:
            raise ValueError("buffers must live in CUDA device memory (use HostExecutor for host buffers)")
        return int(buf.data_ptr())
    raise TypeError(f"unsupported buffer type {type(buf)}")


def _strided_ptr(buf, block, strides, batch) -> int:
    """_ptr of a buffer on a side with strides (dfft_plan_set_strides): a tensor of the block's shape ([batch, X, Y, Z] when
    batched) whose strides are the declared {field, x, y} and 1 along z; dimensions of extent 1 may have any stride"""
    if buf is None or isinstance(buf, int) or not hasattr(buf, "data_ptr"):
        return _ptr(buf)
    shape = (tuple(block) if batch == 1 else (batch, *block))
    want = (tuple(strides[1:]) + (1,)) if batch == 1 else (tuple(strides) + (1,))
    if tuple(buf.shape) != shape:
        raise ValueError(f"a buffer with strides must have the block's shape {shape}, got {tuple(buf.shape)}")
    if any(n > 1 and s != w for n, s, w in zip(buf.shape, buf.stride(), want)):
        raise ValueError(f"buffer strides {tuple(buf.stride())} differ from the plan's {want}")
    if hasattr(buf, "is_cuda") and not buf.is_cuda:
        raise ValueError("buffers must live in CUDA device memory (use HostExecutor for host buffers)")
    return int(buf.data_ptr())


def _stream_ptr(stream) -> int:
    if stream is None:
        return 0
    if isinstance(stream, int):
        return stream
    return int(stream.cuda_stream)


class Comm:
    """Replaces MPI_Comm: one rank per process/GPU, NCCL underneath (src/mpicufft.cpp:42-50)."""

    def __init__(self, rank: int = 0, nranks: int = 1, unique_id: Optional[bytes] = None, device: int = 0):
        h = C.c_void_p()
        idbuf = None
        if nranks > 1:
            if unique_id is None or len(unique_id) != _lib.UNIQUE_ID_BYTES:
                raise ValueError("unique_id of 128 bytes required for nranks > 1")
            idbuf = C.create_string_buffer(unique_id, _lib.UNIQUE_ID_BYTES)
        check(lib().dfft_comm_create(rank, nranks, idbuf, device, C.byref(h)))
        self._h = h
        self.rank, self.size, self.device = rank, nranks, device

    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(_lib.UNIQUE_ID_BYTES)
        check(lib().dfft_get_unique_id(buf))
        return buf.raw

    @classmethod
    def from_torch_distributed(cls, device: Optional[int] = None) -> "Comm":
        """Build the communicator of the current torch.distributed world (rank 0 creates the NCCL id,
        torch broadcasts it — the role MPI_Bcast would play in the reference's launcher)."""
        import torch
        import torch.distributed as dist

        if not dist.is_initialized() or dist.get_world_size() == 1:
            return cls(0, 1, None, torch.cuda.current_device() if device is None else device)
        rank, world = dist.get_rank(), dist.get_world_size()
        box = [cls.unique_id() if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        return cls(rank, world, box[0], torch.cuda.current_device() if device is None else device)

    def destroy(self):
        if self._h:
            lib().dfft_comm_destroy(self._h)
            self._h = None


class MPIcuFFT:
    """Abstract plan (include/mpicufft.hpp:55-105). `precision`: 'double' | 'float' replaces the C++
    template argument; 'half' ('f16', 'float16') and 'bfloat16' ('bf16') make 16-bit plans (C2C and R2C / C2R, power-of-two
    lengths; f32 arithmetic inside the passes, include/dfft.h): their buffers are torch.complex32 / torch.float16 tensors
    (FP16) or torch.bfloat16 tensors with a trailing dimension of 2 on complex sides and plain torch.bfloat16 on real sides
    (BF16), and the output scale is split over the FFT passes (setScale).  `transform`: 'r2c' (the reference's), 'c2c', or the real-to-real 'dct' / 'dst' (type II forward, type III
    inverse, on all three axes; execR2R).  A tuple of three names from 'dct', 'dst', 'r2hc', 'dct1', 'dst1', 'dct4', 'dst4',
    in (x, y, z) order, gives a real-to-real plan with a kind per axis (dfft_plan_create_r2r; 'r2hc': FFTW's R2HC forward,
    HC2R inverse; 'dct1' / 'dst1': DCT-I / DST-I both ways, FFTW's REDFT00 / RODFT00, on axes of 2^k + 1 / 2^k - 1 points;
    'dct4' / 'dst4': DCT-IV / DST-IV both ways, FFTW's REDFT11 / RODFT11, on cell-centred axes of 2^k points, 4..8192, with
    a Neumann wall at one end and a Dirichlet wall at the other), e.g. ("dct1", "r2hc", "r2hc") for a Chebyshev
    wall-normal x axis or ("dct4", "r2hc", "r2hc") for a channel with a no-slip bed and a free-slip lid."""

    _decomp = SLAB_ZY_THEN_X

    def __init__(self, config: Configurations, comm: Optional[Comm] = None, max_world_size: int = -1,
                 precision: str = "double", transform: str = "r2c"):
        self.config = config
        self.comm = comm if comm is not None else Comm()
        if precision in ("double", "f64", "float64"):
            self.precision = F64
        elif precision in ("float", "f32", "float32"):
            self.precision = F32
        elif precision in ("half", "f16", "float16"):
            self.precision = F16
        elif precision in ("bfloat16", "bf16"):
            self.precision = BF16
        else:
            raise ValueError(f"precision must be 'double', 'float', 'half' or 'bfloat16', got {precision!r}")
        self.kinds = None
        if isinstance(transform, tuple):
            if len(transform) != 3 or not all(isinstance(k, str) and k.lower() in _R2R_KINDS for k in transform):
                raise ValueError(f"a per-axis transform is three of 'dct', 'dst', 'r2hc', 'dct1', 'dst1', 'dct4', 'dst4', got {transform!r}")
            self.kinds = tuple(_R2R_KINDS[k.lower()] for k in transform)
            # as the library records it: three DCT (DST) axes are the DCT (DST) plan, every other combination a per-axis one
            uniform = len(set(self.kinds)) == 1 and self.kinds[0] in (DCT, DST)
            self.transform = self.kinds[0] if uniform else R2HC
        elif transform in ("r2c", "R2C"):
            self.transform = R2C
        elif transform in ("c2c", "C2C"):
            self.transform = C2C
        elif transform in ("dct", "DCT"):
            self.transform = DCT
        elif transform in ("dst", "DST"):
            self.transform = DST
        else:
            raise ValueError(f"transform must be 'r2c', 'c2c', 'dct' or 'dst', got {transform!r}")
        self._h = None
        self.initialized = False

    # -- plan ------------------------------------------------------------------------------------
    def initFFT(self, global_size: GlobalSize, partition: Optional[Partition] = None, allocate: bool = True, batch: int = 1,
                inplace: bool = False, transform_axes: Optional[Sequence[bool]] = None, spectral: Optional[Sequence[int]] = None,
                components: int = 1, in_boxes=None, out_boxes=None, in_strides=None, out_strides=None, data: Optional[Sequence[int]] = None,
                signal: Optional[int] = None, factors: Optional[Sequence[int]] = None, natural: bool = False):
        """`batch` (not in the reference): every exec transforms that many fields, back to back in each buffer — a
        contiguous [batch, X, Y, Z] tensor; the getters describe one field (dfft_plan_create_batched).
        `inplace` (dfft_plan_create_inplace): every exec gets the same buffer twice and overwrites its input; fields are
        getDomainSize() bytes apart.  R2C / C2R use padded real rows: with buf a complex [X, Y, Nz/2+1] tensor, pass
        torch.view_as_real(buf).view(X, Y, Nz + 2) as the real side.
        `transform_axes` (x, y, z): setTransformAxes right after creation, e.g. (False, True, True) keeps x.
        `spectral` (kx, ky, kz) (dfft_plan_create_padded): a padded plan, global_size the physical grid and (kx, ky, kz) the
        spectrum it keeps — the forward stores only those modes, the inverse zero-pads them (the 3/2 dealiasing rule).
        `components` C (dfft_plan_create_interleaved): every grid point holds C consecutive values, each component
        transformed on its own — buffers are [X, Y, Z, C] tensors ([B, X, Y, Z, C] with a batch), reals on the real side
        of R2C / C2R; C > 1 plans are C2C or R2C / C2R, out of place and not padded.
        `in_boxes` / `out_boxes` (dfft_plan_create_boxes): one box ((lx, ly, lz), (hx, hy, hz)) per rank, in rank order, of the
        physical grid and of the output grid (z extent Nz/2 + 1 for R2C); each rank's buffer on that side is its box, a dense
        [hx-lx, hy-ly, hz-lz] tensor, and the exec redistributes on the GPU.  None keeps the natural layout.  Box plans are
        out of place, not padded, with one component and one transform for all axes.
        `in_strides` / `out_strides` (field, x, y) (dfft_plan_set_strides): the buffers of the physical side / of the output
        of d = 3 lie inside larger arrays, e.g. the interior A[h:-h, h:-h, h:-h] of a field with ghost cells, whose strides
        these are (torch's .stride(), in elements: reals on the real side of R2C / C2R and for R2R plans); such a side then
        takes exactly those non-contiguous tensors.  None keeps a side dense.
        `data` (mx, my, mz) (dfft_plan_create_pruned): a pruned plan, global_size the transform grid and the field an
        [mx, my, mz] block at the origin, zero beyond — the forward reads only the block, the inverse stores only it (the
        doubled grid of free-space solvers).  The physical side of every exec is this rank's m-block; combines with
        `spectral`.  Pruned plans are out of place, C2C or R2C, with one component and no boxes or strides.
        `signal` n (dfft_plan_create_1d, MPIcuFFT_Slab only): a distributed 1D C2C transform of one n-point signal, seen as
        the grid (N1, N2, N3) = `factors` (None: the library's balanced choice, getFactors()) with global_size None.  Each
        rank's buffers are its x-slab [in_size[0], N2, N3] of that grid on both sides, the forward output in scrambled order
        (frequency k at [k % N1][(k // N1) % N2][k // (N1 N2)]); 1D plans are C2C, out of place, batch 1, without
        partition, strides or kept axes.
        `natural` (with `signal`, dfft_plan_create_1d_natural): the forward output in natural order instead: each rank's out
        is its chunk [out_size[0], N2, N1] of the spectrum, frequencies getOutStart()[0] * N1 * N2 on, k increasing (flat
        index k - that start); the inverse takes that chunk.  N3 must then be at least the rank count as well."""
        if signal is not None:
            if self._decomp != SLAB_ZY_THEN_X:
                raise ValueError("1D plans are slab plans (MPIcuFFT_Slab)")
            if self.transform != C2C or global_size is not None or partition is not None or batch != 1 or not allocate or \
                    transform_axes is not None or in_strides is not None or out_strides is not None:
                raise ValueError("1D plans are C2C, out of place and allocated, batch 1, with no global_size, partition, strides or "
                                 "transform_axes")
        elif factors is not None:
            raise ValueError("factors belong to a 1D plan (signal=n)")
        elif natural:
            raise ValueError("natural belongs to a 1D plan (signal=n)")
        elif global_size is None:
            raise RuntimeError("GlobalSize or Partition not initialized!")
        cfg = _lib.dfft_config(int(self.config.cuda_aware), int(self.config.warmup_rounds), int(self.config.comm_method),
                               int(self.config.send_method),
                               self.config.benchmark_dir.encode() if self.config.benchmark_dir else None,
                               int(self.config.comm_method2), int(self.config.send_method2))
        p1 = partition.P1 if partition is not None else self.comm.size
        p2 = partition.P2 if partition is not None else 1
        if self._decomp == PENCIL and partition is None:
            raise RuntimeError("GlobalSize or Partition not initialized!")
        h = C.c_void_p()
        L, head, n = lib(), (self.comm._h, C.byref(cfg), self._decomp, self.precision), (global_size.Nx, global_size.Ny, global_size.Nz) if global_size else ()
        tail = (batch, 1 if allocate else 0, C.byref(h))

        def sizes(v):
            return None if v is None else (C.c_size_t * 3)(*(int(k) for k in v))

        def xyz(v):
            x, y, z = (int(k) for k in v)
            return x, y, z

        def flat(boxes):
            if boxes is None:
                return None
            boxes = list(boxes)
            if len(boxes) != self.comm.size:
                raise ValueError(f"{len(boxes)} boxes for {self.comm.size} ranks")
            vals = [int(v) for lo, hi in boxes for v in (*lo, *hi)]
            if len(vals) != 6 * self.comm.size:
                raise ValueError("a box is ((lx, ly, lz), (hx, hy, hz))")
            return (C.c_size_t * len(vals))(*vals)
        # The creators, in the order they are chosen: (keyword, given, the other keywords it takes, why it refuses the rest,
        # call).  The first one given makes the plan, and any other keyword given that it does not take raises ValueError
        # before the library is called.
        creators = (
            ("natural", signal is not None and bool(natural), ("signal",),
             "1D plans are out of place and C2C, with one component, no boxes and the whole grid",
             lambda: L.dfft_plan_create_1d_natural(self.comm._h, C.byref(cfg), self.precision, int(signal), sizes(factors), C.byref(h))),
            ("signal", signal is not None, (), "1D plans are out of place and C2C, with one component, no boxes and the whole grid",
             lambda: L.dfft_plan_create_1d(self.comm._h, C.byref(cfg), self.precision, int(signal), sizes(factors), C.byref(h))),
            ("data", data is not None, ("spectral",), "pruned plans are out of place, C2C or R2C, with one component and no boxes",
             lambda: L.dfft_plan_create_pruned(*head, self.transform, *n, sizes(data), sizes(spectral), p1, p2, *tail)),
            ("boxes", in_boxes is not None or out_boxes is not None, (),
             "box plans are out of place, not padded, with one component and one transform kind for all axes",
             lambda: L.dfft_plan_create_boxes(*head, self.transform, *n, p1, p2, flat(in_boxes), flat(out_boxes), *tail)),
            ("components", components != 1, (), "interleaved plans are out of place and not padded",
             lambda: L.dfft_plan_create_interleaved(*head, self.transform, *n, p1, p2, int(components), *tail)),
            ("spectral", spectral is not None, (), "padded plans are out of place and C2C or R2C",
             lambda: L.dfft_plan_create_padded(*head, self.transform, *n, *xyz(spectral), p1, p2, *tail)),
            ("kinds", self.kinds is not None, ("inplace",), None,
             lambda: L.dfft_plan_create_r2r(*head, (C.c_int * 3)(*self.kinds), *n, p1, p2, batch, 1 if inplace else 0, *tail[1:])),
            ("inplace", bool(inplace), (), None, lambda: L.dfft_plan_create_inplace(*head, self.transform, *n, p1, p2, *tail)),
            (None, True, (), None, lambda: L.dfft_plan_create(*head, self.transform, *n, p1, p2, *tail[1:]) if batch == 1 else
             L.dfft_plan_create_batched(*head, self.transform, *n, p1, p2, *tail)),
        )
        keyword, _, takes, refusal, create = next(c for c in creators if c[1])
        if any(c[0] not in (keyword, *takes) for c in creators[:-1] if c[1]):
            raise ValueError(refusal)
        if batch < 1:
            raise ValueError("batch must be at least 1")
        check(create())
        self._h = h
        if signal is not None:
            global_size = GlobalSize(*self.getFactors())
        self.global_size = global_size
        self.initialized = True
        self._strides = (None, None)
        try:
            if in_strides is not None or out_strides is not None:
                self.setStrides(in_strides, out_strides)
            if transform_axes is not None:
                self.setTransformAxes(*transform_axes)
        except Exception:
            self.destroy()
            self.initialized = False
            raise

    def setStrides(self, in_strides=None, out_strides=None):
        """{field, x, y} strides of the caller's arrays on the physical side (in) and on the output of d = 3 (out), z
        contiguous (dfft_plan_set_strides).  Only before the first exec, tune or describe; every rank calls it with its own
        values, or none does."""
        self._need()

        def arr(s):
            return None if s is None else (C.c_longlong * 3)(*(int(v) for v in s))
        check(lib().dfft_plan_set_strides(self._h, arr(in_strides), arr(out_strides)))
        self._strides = (None if in_strides is None else tuple(int(v) for v in in_strides),
                         None if out_strides is None else tuple(int(v) for v in out_strides))

    def getStrides(self):
        """((field, x, y) of the physical side, (field, x, y) of the output), the dense ones for a side without strides"""
        self._need()
        i, o = (C.c_longlong * 3)(), (C.c_longlong * 3)()
        check(lib().dfft_plan_get_strides(self._h, i, o))
        return tuple(i), tuple(o)

    def _bufs(self, out, in_, physical_in: bool, d: int):
        """(out, in) pointers of an exec; physical_in: `in_` is the physical side (forward), else `out` is"""
        phys, spec = getattr(self, "_strides", (None, None))
        spec = spec if d == 3 else None
        batch = self.getBatch() if phys is not None or spec is not None else 1

        def one(buf, physical):
            s = phys if physical else spec
            if s is None:
                return _ptr(buf)
            return _strided_ptr(buf, self.getInSize() if physical else self.getOutSize(), s, batch)
        return one(out, not physical_in), one(in_, physical_in)

    def setTransformAxes(self, x: bool = True, y: bool = True, z: bool = True):
        """Transform (True) or keep (False) each axis (dfft_plan_set_transform_axes).  A kept axis is redistributed as a
        transformed one would be but its values are not transformed: (False, True, True) transforms z and y and returns
        x whole on every rank, in the output layout, for a solve along x.  Only before the first exec, tune or describe;
        local to this rank (set the same values on every rank).  R2C plans must transform z."""
        self._need()
        check(lib().dfft_plan_set_transform_axes(self._h, (C.c_int * 3)(int(bool(x)), int(bool(y)), int(bool(z)))))

    def getTransformAxes(self):
        """(x, y, z): True where the axis is transformed."""
        self._need()
        t = (C.c_int * 3)()
        check(lib().dfft_plan_get_transform_axes(self._h, t))
        return tuple(bool(v) for v in t)

    def setWorkArea(self, device=None, host=None):
        check(lib().dfft_set_work_area(self._h, _ptr(device), _ptr(host)))

    def destroy(self):
        if self._h:
            lib().dfft_plan_destroy(self._h)
            self._h = None

    # -- exec ------------------------------------------------------------------------------------
    def _need(self):
        if not self.initialized:
            raise RuntimeError("plan not initialised (call initFFT)")

    def execR2C(self, out, in_, d: int = 3, stream=None):
        """Real-to-complex transform.  With `stream` the exec is only enqueued there (dfft_exec_r2c_async); such a call may
        be captured into a CUDA graph (torch.cuda.graph) on one-rank plans once this direction has run eagerly
        (INTEGRATION.md section 4)."""
        self._need()
        if stream is not None:
            if d != 3:
                raise ValueError("async partial transforms are not exposed")
            return check(lib().dfft_exec_r2c_async(self._h, *self._bufs(out, in_, True, 3), _stream_ptr(stream)))
        if d == 3:
            return check(lib().dfft_exec_r2c(self._h, *self._bufs(out, in_, True, 3)))
        return check(lib().dfft_exec_r2c_partial(self._h, *self._bufs(out, in_, True, d), d))

    def execC2R(self, out, in_, d: int = 3, stream=None):
        """Complex-to-real transform; `stream` as for execR2C, capturable the same way."""
        self._need()
        if stream is not None:
            if d != 3:
                raise ValueError("async partial transforms are not exposed")
            return check(lib().dfft_exec_c2r_async(self._h, *self._bufs(out, in_, False, 3), _stream_ptr(stream)))
        if d == 3:
            return check(lib().dfft_exec_c2r(self._h, *self._bufs(out, in_, False, 3)))
        return check(lib().dfft_exec_c2r_partial(self._h, *self._bufs(out, in_, False, d), d))

    def execC2C(self, out, in_, direction: int = FORWARD, d: int = 3, stream=None):
        """Complex transform (not in the reference; BASELINE configs 1-4 need it).  `stream` as for execR2C, capturable
        the same way."""
        self._need()
        if stream is not None:
            if d != 3:
                raise ValueError("async partial transforms are not exposed")
            return check(lib().dfft_exec_c2c_async(self._h, *self._bufs(out, in_, direction <= 0, 3), direction, _stream_ptr(stream)))
        if d == 3:
            return check(lib().dfft_exec_c2c(self._h, *self._bufs(out, in_, direction <= 0, 3), direction))
        return check(lib().dfft_exec_c2c_partial(self._h, *self._bufs(out, in_, direction <= 0, d), direction, d))

    def execR2R(self, out, in_, direction: int = FORWARD, d: int = 3, stream=None):
        """Real-to-real transform of a 'dct' / 'dst' or per-axis plan (not in the reference): FORWARD is type II (R2HC on
        'r2hc' axes), INVERSE type III (HC2R), all unnormalised like scipy.fft.dct / dst(norm=None); 'dct1' / 'dst1' axes
        run DCT-I / DST-I (type=1) and 'dct4' / 'dst4' axes DCT-IV / DST-IV (type=4) in both directions.  Real [x][y][z] buffers.  `stream` as for execR2C, capturable the
        same way."""
        self._need()
        if stream is not None:
            if d != 3:
                raise ValueError("async partial transforms are not exposed")
            return check(lib().dfft_exec_r2r_async(self._h, *self._bufs(out, in_, direction <= 0, 3), direction, _stream_ptr(stream)))
        if d == 3:
            return check(lib().dfft_exec_r2r(self._h, *self._bufs(out, in_, direction <= 0, 3), direction))
        return check(lib().dfft_exec_r2r_partial(self._h, *self._bufs(out, in_, direction <= 0, d), direction, d))

    def getR2RKinds(self):
        """(x, y, z) kinds of a real-to-real plan: DCT, DST, R2HC, DCT1, DST1, DCT4 or DST4 each (dfft_plan_get_r2r_kinds)."""
        self._need()
        k = (C.c_int * 3)()
        check(lib().dfft_plan_get_r2r_kinds(self._h, k))
        return tuple(k)

    def wait(self):
        return check(lib().dfft_plan_wait(self._h))

    def tune(self, out, in_, direction: int = FORWARD, reps: int = 3) -> str:
        """Plan-time measurement: try the sequential and the overlapped schedules on these buffers and keep the fastest
        (collective).  Returns the report string."""
        self._need()
        check(lib().dfft_plan_tune(self._h, *self._bufs(out, in_, direction <= 0, 3), 1 if direction > 0 else 0, reps))
        return (lib().dfft_plan_tune_report(self._h) or b"").decode()

    # -- getters ---------------------------------------------------------------------------------
    def _triple(self, fn, *a):
        v = (C.c_size_t * 3)()
        check(fn(self._h, *a, v))
        return [int(x) for x in v]

    def getInSize(self): return self._triple(lib().dfft_get_in_size)
    def getInStart(self): return self._triple(lib().dfft_get_in_start)
    def getOutSize(self): return self._triple(lib().dfft_get_out_size)
    def getOutStart(self): return self._triple(lib().dfft_get_out_start)
    def getPartialSize(self, d): return self._triple(lib().dfft_get_partial_size, d)
    def getPartialStart(self, d): return self._triple(lib().dfft_get_partial_start, d)
    def getDomainSize(self): return int(lib().dfft_get_domain_size(self._h))
    def getSpectralSize(self): return self._triple(lib().dfft_plan_get_spectral_size)
    def getDataSize(self): return self._triple(lib().dfft_plan_get_data_size)
    def getFactors(self): return self._triple(lib().dfft_plan_get_1d_factors)
    def getBatch(self): return int(lib().dfft_get_batch(self._h))
    def getComponents(self): return int(lib().dfft_get_components(self._h))
    def isInPlace(self): return bool(lib().dfft_plan_is_inplace(self._h))
    def getWorkSizeDevice(self): return int(lib().dfft_get_work_size_device(self._h))
    def getWorkSizeHost(self): return int(lib().dfft_get_work_size_host(self._h))
    def getWorkAreaDevice(self): return lib().dfft_get_work_area_device(self._h)
    def getWorkAreaHost(self): return None
    def getRank(self): return int(lib().dfft_get_rank(self._h))
    def getWorldSize(self): return int(lib().dfft_get_world_size(self._h))

    # -- output scale (not in the reference) ------------------------------------------------------
    def setScale(self, forward: float = 1.0, inverse: float = 1.0):
        """Multiply every output value of forward / inverse execs by these scales, inside the kernel that stores them
        (dfft_plan_set_scale).  With N the product of the transformed lengths: torch's norm="backward" is (1, 1/N),
        "ortho" (1/sqrt(N), 1/sqrt(N)), "forward" (1/N, 1).  Local to this rank: set the same values on every rank.
        A CUDA graph keeps the scale it was captured with; run each direction eagerly once before capturing again."""
        check(lib().dfft_plan_set_scale(self._h, float(forward), float(inverse)))

    def getScale(self):
        """(forward, inverse) output scales."""
        f, i = C.c_double(), C.c_double()
        check(lib().dfft_plan_get_scale(self._h, C.byref(f), C.byref(i)))
        return f.value, i.value

    # -- spectral weights (not in the reference) --------------------------------------------------
    def setWeights(self, wx=None, wy=None, wz=None):
        """Per-axis spectral weights (dfft_plan_set_weights): forward execs return W * F(x), inverse ones F^-1(W * X), with
        W[kx, ky, kz] = wx[kx] * wy[ky] * wz[kz] multiplied inside the FFT passes.  Each is None (all ones) or a contiguous
        1-D complex128 (double plans) / complex64 (float plans) CUDA tensor on the plan's device, as long as the axis's
        spectral extent: getSpectralSize(), Kz // 2 + 1 on z for R2C / C2R.  The plan reads the tensors at every exec and
        keeps references to them; rewrite them in place between execs, or call again to re-point.  The first call must come
        before the first exec, tune or describe.  C2R plans: make W Hermitian (e.g. zero the Nyquist entry of i k)."""
        import torch

        self._need()
        ptrs = (C.c_void_p * 3)()
        want = {F64: torch.complex128, F32: torch.complex64}.get(self.precision)
        if want is None:  # 16-bit plans: the library's refusal
            check(lib().dfft_plan_set_weights(self._h, ptrs))
        k = list(self.getSpectralSize())
        if self.transform == R2C:
            k[2] = k[2] // 2 + 1
        for a, (name, w) in enumerate((("wx", wx), ("wy", wy), ("wz", wz))):
            if w is None:
                continue
            if not isinstance(w, torch.Tensor) or w.dtype != want:
                raise TypeError(f"{name} must be a {want} tensor")
            if not w.is_cuda or w.device.index != self.comm.device:
                raise ValueError(f"{name} must be on cuda:{self.comm.device}, the plan's device")
            if w.dim() != 1 or not w.is_contiguous() or w.numel() != k[a]:
                raise ValueError(f"{name} must be a contiguous 1-D tensor of {k[a]} values, got shape {tuple(w.shape)}")
            ptrs[a] = w.data_ptr()
        check(lib().dfft_plan_set_weights(self._h, ptrs))
        self._weights = (wx, wy, wz)  # the plan reads these at every exec: keep them alive

    def getWeights(self):
        """(wx, wy, wz): the tensors given to the last setWeights, None where none was given."""
        self._need()
        return getattr(self, "_weights", (None, None, None))

    # -- timer -----------------------------------------------------------------------------------
    def enableTimer(self, on: bool = True):
        check(lib().dfft_timer_enable(self._h, 1 if on else 0))

    def phaseTimes(self):
        n = lib().dfft_get_phase_count(self._h)
        ms = (C.c_double * max(n, 1))()
        n = check(lib().dfft_get_phase_times(self._h, ms, n))
        return [(lib().dfft_get_phase_name(self._h, i).decode(), float(ms[i])) for i in range(n)]

    def stepTimes(self):
        """[(label, ms)] per launched step of the last timed exec."""
        n = lib().dfft_get_step_count(self._h)
        ms = (C.c_double * max(n, 1))()
        n = check(lib().dfft_get_step_times(self._h, ms, n))
        return [(lib().dfft_get_step_label(self._h, i).decode(), float(ms[i])) for i in range(n)]

    def timeline(self):
        """[(label, stream, begin_ms, end_ms)] of the last timed exec — every step on its own plan stream."""
        cap = 256
        b = (C.c_double * cap)(); e = (C.c_double * cap)(); st = (C.c_int * cap)()
        n = check(lib().dfft_get_timeline(self._h, b, e, st, cap))
        return [(lib().dfft_get_timeline_label(self._h, i).decode(), int(st[i]), float(b[i]), float(e[i])) for i in range(min(n, cap))]

    def lastBreakdown(self):
        f, x, t = C.c_double(), C.c_double(), C.c_double()
        check(lib().dfft_get_last_breakdown(self._h, C.byref(f), C.byref(x), C.byref(t)))
        return {"fft_ms": f.value, "exchange_ms": x.value, "total_ms": t.value}

    def lastLaunchCount(self):
        return int(lib().dfft_get_last_launch_count(self._h))


class MPIcuFFT_Slab(MPIcuFFT):
    """2D (y,z) FFT -> transpose (x split -> y split) -> 1D x FFT. include/mpicufft_slab.hpp."""
    _decomp = SLAB_ZY_THEN_X


class MPIcuFFT_Slab_Z_Then_YX(MPIcuFFT):
    """1D z FFT -> transpose (x split -> z split) -> 2D (y,x) FFT. include/mpicufft_slab_z_then_yx.hpp."""
    _decomp = SLAB_Z_THEN_YX


class MPIcuFFT_Pencil(MPIcuFFT):
    """z FFT -> transpose -> y FFT -> transpose -> x FFT on a P1 x P2 grid. include/mpicufft_pencil.hpp."""
    _decomp = PENCIL

    def initFFT(self, global_size, partition=None, allocate=True, batch=1, inplace=False, transform_axes=None, spectral=None, components=1,
                in_boxes=None, out_boxes=None, in_strides=None, out_strides=None, data=None):
        if partition is None or global_size is None:
            raise RuntimeError("GlobalSize or Partition not initialized!")
        if partition.P1 * partition.P2 != self.comm.size:
            raise RuntimeError("Invalid Input Partition!")
        self.partition = partition
        super().initFFT(global_size, partition, allocate, batch, inplace, transform_axes, spectral, components, in_boxes, out_boxes, in_strides,
                        out_strides, data)

    def getPartitionDimensions(self):
        """(input_dim, transposed_dim, output_dim), each a dict with size_x/y/z and start_x/y/z lists
        (Partition_Dimensions, params.hpp:58-81; mpicufft_pencil.hpp:112-116)."""
        from .params import partition_sizes
        g, p = self.global_size, self.partition
        nzc = g.Nz // 2 + 1 if self.transform == R2C else g.Nz

        def dims(nx_parts, ny_parts, nz_parts, nz):
            d = {}
            for ax, n, parts in (("x", g.Nx, nx_parts), ("y", g.Ny, ny_parts), ("z", nz, nz_parts)):
                d[f"size_{ax}"], d[f"start_{ax}"] = partition_sizes(n, parts)
            return d
        return dims(p.P1, p.P2, 1, g.Nz), dims(p.P1, 1, p.P2, nzc), dims(1, p.P1, p.P2, nzc)


# "Realigned" (Opt1) classes of the reference — include/mpicufft_slab_opt1.hpp, mpicufft_slab_z_then_yx_opt1.hpp,
# mpicufft_pencil_opt1.hpp: same results and output layouts as the default classes; the transposing store they add is
# always fused into the FFT passes here, so they are aliases.
MPIcuFFT_Slab_Opt1 = MPIcuFFT_Slab
MPIcuFFT_Slab_Z_Then_YX_Opt1 = MPIcuFFT_Slab_Z_Then_YX
MPIcuFFT_Pencil_Opt1 = MPIcuFFT_Pencil


def layout(decomp: int, transform: int, nx: int, ny: int, nz: int, p1: int, p2: int, rank: int, which: int):
    """Geometry of any rank without a device (dfft_layout): which = 0 in, 1 after z, 2 after z,y, 3 out."""
    size = (C.c_size_t * 3)()
    start = (C.c_size_t * 3)()
    check(lib().dfft_layout(decomp, transform, nx, ny, nz, p1, p2, rank, which, size, start))
    return [int(x) for x in size], [int(x) for x in start]


def fft1d_contig(precision: int, kind: int, direction: int, n: int, lines: int, out, out_pitch: int, in_, in_pitch: int, stream=None):
    check(lib().dfft_fft1d_contig(precision, kind, direction, n, lines, _ptr(out), out_pitch, _ptr(in_), in_pitch, _stream_ptr(stream)))


def fft1d_strided(precision: int, direction: int, a: int, n: int, b: int, out, in_, stream=None):
    check(lib().dfft_fft1d_strided(precision, direction, a, n, b, _ptr(out), _ptr(in_), _stream_ptr(stream)))


def fft1d_r2r(precision: int, transform: int, direction: int, n: int, a: int, b: int, out, in_, stream=None):
    """DCT / DST / R2HC (transform DCT, DST or R2HC; FORWARD type II or R2HC, INVERSE type III or HC2R) along the middle
    axis of a dense real [a][n][b] array, b contiguous; out may be in_.  DCT1 / DST1: DCT-I / DST-I in both directions,
    n = 2^k + 1 (DCT-I, 3..8193) or 2^k - 1 (DST-I, 3..8191).  DCT4 / DST4: DCT-IV / DST-IV in both directions, n = 2^k
    in 4..8192."""
    check(lib().dfft_fft1d_r2r(precision, transform, direction, n, a, b, _ptr(out), _ptr(in_), _stream_ptr(stream)))


def fft1d_general(precision: int, direction: int, n: int, a0: int, a1: int, b: int, out, out_strides, in_, in_strides, stream=None):
    """Batched C2C along n over a general view: element (i0,i1,n,ib) at i0*s[0] + i1*s[1] + n*s[2] + ib."""
    os_ = (C.c_longlong * 3)(*out_strides)
    is_ = (C.c_longlong * 3)(*in_strides)
    check(lib().dfft_fft1d_general(precision, direction, n, a0, a1, b, _ptr(out), os_, _ptr(in_), is_, _stream_ptr(stream)))
