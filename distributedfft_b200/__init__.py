"""distributedfft_b200 — H100-native distributed 3D FFT behind the plan/execute surface of
eggersn/DistributedFFT (the package keeps its original name).  The compute path is libdfft.so (hand-written sm_90a CUDA + NCCL / NVLink peer
stores); this package is the thin host-side mirror of the reference's classes over its C ABI."""
from .params import (CommunicationMethod, Configurations, GlobalSize, Partition, Pencil_Partition, SendMethod,
                     Slab_Partition, partition_sizes)
from .host import HostExecutor, gpu_local_cpus, numa_local, pinned_empty
from .mpicufft import (BF16, C2C, DCT, DCT1, DCT4, DST, DST1, DST4, F16, F32, F64, FORWARD, INVERSE, PENCIL, R2C, R2HC, SLAB_Z_THEN_YX, SLAB_ZY_THEN_X, Comm, MPIcuFFT,
                       MPIcuFFT_Pencil, MPIcuFFT_Pencil_Opt1, MPIcuFFT_Slab, MPIcuFFT_Slab_Opt1, MPIcuFFT_Slab_Z_Then_YX,
                       MPIcuFFT_Slab_Z_Then_YX_Opt1, fft1d_contig, fft1d_general, fft1d_r2r, fft1d_strided, layout)

__all__ = [n for n in dir() if not n.startswith("_")]
