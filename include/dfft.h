/* dfft.h — C ABI of the H100-native distributed 3D FFT (libdfft.so).
 *
 * Drop-in boundary for the plan/execute surface of eggersn/DistributedFFT. The reference exposes a C++
 * class hierarchy, one object per MPI rank, one rank per GPU:
 *     MPIcuFFT<T>            /root/reference/include/mpicufft.hpp:55-105
 *     MPIcuFFT_Slab<T>       /root/reference/include/mpicufft_slab.hpp:88-125
 *     MPIcuFFT_Slab_Z_Then_YX<T>  /root/reference/include/mpicufft_slab_z_then_yx.hpp
 *     MPIcuFFT_Pencil<T>     /root/reference/include/mpicufft_pencil.hpp:71-122
 * This header is what a binding of those classes would link against: plain pointers and sizes, no C++
 * or torch types.  include/dfft.hpp re-creates the reference's class and method names on top of it.
 *
 * Process model: identical to the reference — one process (rank) per GPU.  MPI_Comm is replaced by
 * dfft_comm_t, which wraps an NCCL communicator; the 128-byte unique id is produced on rank 0 by
 * dfft_get_unique_id and broadcast by whatever launcher the caller already has (MPI_Bcast,
 * torch.distributed.broadcast_object_list, a file).
 *
 * All device pointers are CUDA device pointers on the communicator's device.  Every function returns
 * DFFT_SUCCESS (0) or a negative dfft_status; dfft_last_error_string() describes the last failure of
 * the calling thread.  (The reference prints and calls exit(EXIT_FAILURE) —
 * /root/reference/src/slab/default/mpicufft_slab.cpp:23-29 — the C++ shim keeps that behaviour.)
 */
#ifndef DFFT_H_
#define DFFT_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DFFT_VERSION 100
#define DFFT_UNIQUE_ID_BYTES 128

typedef enum {
    DFFT_SUCCESS = 0,
    DFFT_ERR_INVALID = -1,     /* bad argument / unsupported size */
    DFFT_ERR_CUDA = -2,        /* CUDA runtime failure */
    DFFT_ERR_NCCL = -3,        /* NCCL failure */
    DFFT_ERR_STATE = -4,       /* plan not initialised / no work area */
    DFFT_ERR_UNSUPPORTED = -5, /* valid request this build cannot serve */
    DFFT_ERR_PEER = -6,        /* peer memory mapping (CUDA IPC) unavailable */
    DFFT_ERR_TIMEOUT = -7      /* a device-side rendezvous timed out */
} dfft_status;

/* enum CommunicationMethod {Peer2Peer, All2All}  — /root/reference/include/params.hpp:83
 *   Peer2Peer: the FFT kernels store straight into the peers' receive buffers over NVLink
 *              (CUDA-IPC mapped peer memory), no pack, no send buffer, no unpack.
 *   All2All:   the FFT kernels store into per-destination send slots, NCCL grouped send/recv
 *              (all-to-all-v) moves them, the next FFT pass gathers from the receive slots. */
typedef enum { DFFT_PEER2PEER = 0, DFFT_ALL2ALL = 1 } dfft_comm_method;
/* enum SendMethod {Sync, Streams, MPI_Type} — /root/reference/include/params.hpp:84.
 * Accepted for source compatibility; Streams selects the chunk-pipelined schedule where available,
 * MPI_Type is treated like Sync (there is never a separate pack step to elide). */
typedef enum { DFFT_SEND_SYNC = 0, DFFT_SEND_STREAMS = 1, DFFT_SEND_MPI_TYPE = 2 } dfft_send_method;

/* struct Configurations — /root/reference/include/params.hpp:85-93 (same fields, same order). */
typedef struct {
    int cuda_aware;            /* kept for the CSV file name; device buffers are always used */
    int warmup_rounds;         /* execs whose phase times are not recorded */
    int comm_method;           /* dfft_comm_method, first (or only) transposition */
    int send_method;           /* dfft_send_method */
    const char* benchmark_dir; /* where the phase-timer CSV goes; NULL = no CSV */
    int comm_method2;          /* pencil: second transposition */
    int send_method2;
} dfft_config;

/* Which reference class the plan stands for. */
typedef enum {
    DFFT_SLAB_ZY_THEN_X = 0, /* MPIcuFFT_Slab: 2D (y,z) FFT, transpose x-split -> y-split, 1D x FFT */
    DFFT_SLAB_Z_THEN_YX = 1, /* MPIcuFFT_Slab_Z_Then_YX: 1D z FFT, transpose x-split -> z-split, 2D (y,x) */
    DFFT_PENCIL = 2          /* MPIcuFFT_Pencil: z FFT, transpose, y FFT, transpose, x FFT on a P1 x P2 grid */
} dfft_decomp;

typedef enum { DFFT_F32 = 0, DFFT_F64 = 1, DFFT_F16 = 2, DFFT_BF16 = 3 } dfft_prec; /* cuFFT<float> / cuFFT<double>, include/cufft.hpp:22-60 */
/* DFFT_F16 / DFFT_BF16 (not in the reference): 16-bit plans.  Every caller buffer, work-area slot, peer store and NCCL
 * message holds 16-bit values; every pass widens them to float exactly, runs the f32 pass arithmetic with the f32 tables
 * and rounds once, to nearest even, as it stores.  Each pass moves half the bytes of the f32 plan.
 *   - A complex element is a pair (re, im) of IEEE binary16 (DFFT_F16, torch.complex32) or bfloat16 (DFFT_BF16) numbers,
 *     4 bytes; the real side of R2C / C2R holds 2-byte reals.  dfft_get_domain_size, dfft_get_work_size_device and the
 *     batch distances follow: half those of the F32 plan of the same geometry (slots rounded up to 256 bytes).  Partitions,
 *     dfft_layout and every extent getter are unchanged.
 *   - dfft_plan_create, dfft_plan_create_batched and dfft_plan_create_inplace take them, for C2C and R2C / C2R with the
 *     power-of-two lengths of f32 plans; every decomposition, Peer2Peer and All2All, partial d, batches, in place,
 *     dfft_plan_set_transform_axes, the timer, dfft_plan_describe, dfft_debug_run_step and graph capture of one-rank
 *     _async execs work as on f32 plans.  They always run the sequential schedule (dfft_plan_tune has one candidate).
 *   - DFFT_ERR_UNSUPPORTED: other lengths, DFFT_DCT / DFFT_DST and dfft_plan_create_r2r, dfft_plan_create_padded, _pruned,
 *     _interleaved and _boxes, and dfft_plan_set_strides.  A precision outside 0..3: DFFT_ERR_INVALID.
 *   - dfft_fft1d_contig, _strided and _general take them; dfft_fft1d_r2r returns DFFT_ERR_UNSUPPORTED.
 *   - Output scale (dfft_plan_set_scale): a direction's scale s is split over the FFT passes of the exec, so that no
 *     intermediate overflows that the result would not.  With L = sum of log2 n_a over the axes the exec transforms (log2 Nz
 *     for the R2C z axis), the pass over axis a multiplies each value it stores by f_a = float(|s|^(log2 n_a / L)) before
 *     rounding it, and the last FFT pass of the exec also carries the sign of s.  s = 1 runs unscaled; s = 1/N gives
 *     f_a = 1/n_a exactly.  Copy passes of kept axes and execs that transform no axis never scale.  So the f32 / f64 rule
 *     "the output is the unscaled output times s, bit for bit" does not hold here.  FP16 tops out at 65504: an
 *     unnormalised forward of a large grid (a 512^3 field with a non-zero mean) overflows to inf; BF16 has the range of
 *     FP32.  Use (1/N, 1) or (1/sqrt(N), 1/sqrt(N)) with FP16.  dfft_plan_describe lists "precision" ("f16" / "bf16") and
 *     each pass's f_a != 1 as "factor". */

/* The reference only offers real<->complex (execR2C/execC2R).  DFFT_C2C plans add the complex
 * transform the benchmark configurations name; the z extent of every complex array is then Nz instead
 * of Nz/2+1. */
typedef enum { DFFT_R2C = 0, DFFT_C2C = 1, DFFT_DCT = 2, DFFT_DST = 3, DFFT_R2HC = 4 } dfft_transform;
/* DFFT_DCT / DFFT_DST plans (not in the reference; cuFFT has neither, FFTW calls them REDFT10 / REDFT01 and RODFT10 /
 * RODFT01): real-to-real transforms, the same kind along all three axes, for spectral solvers with Neumann (DCT) or
 * Dirichlet (DST) boundaries.  With N the axis length:
 *   forward, type II:   DCT  y_k = 2 sum_n x_n cos(pi k (2n+1) / 2N)      DST  y_k = 2 sum_n x_n sin(pi (k+1)(2n+1) / 2N)
 *   inverse, type III:  DCT  y_k = x_0 + 2 sum_{n>=1} x_n cos(pi n (2k+1) / 2N)
 *                       DST  y_k = (-1)^k x_{N-1} + 2 sum_{n<N-1} x_n sin(pi (n+1)(2k+1) / 2N)
 * exactly scipy.fft.dct / dst(type=2 | 3, norm=None).  Both directions are unnormalised: a round trip scales by
 * 8 Nx Ny Nz (partial transforms: 2^d times the product of the first d lengths).
 *   - Buffers are real [x][y][z], z contiguous, with the partition and the getters of a C2C plan (the z extent is Nz
 *     everywhere); dfft_get_domain_size counts bytes of reals.
 *   - Lengths: powers of two in [2, 8192] per axis; others return DFFT_ERR_UNSUPPORTED.
 *   - Every decomposition with Peer2Peer and All2All, partial d, batches, in-place plans, dfft_plan_set_scale, graph
 *     capture of one-rank _async execs, the timer and dfft_plan_describe work as for C2C plans.
 *   - Execs: dfft_exec_r2r*; the R2C / C2R / C2C execs return DFFT_ERR_INVALID on these plans, and dfft_exec_r2r* on
 *     others.
 *   - The sequential schedule always runs, also with send_method Streams (dfft_plan_tune has one candidate). */
/* DFFT_R2HC (not in the reference; FFTW's R2HC / HC2R): the real DFT of a periodic axis in FFTW's halfcomplex format, a
 * kind only for dfft_plan_create_r2r and dfft_fft1d_r2r (dfft_plan_create* return DFFT_ERR_INVALID for transform 4).
 * Forward (R2HC) of N reals x, with X = DFT_N(x) = sum_n x_n exp(-2 pi i k n / N):
 *   hc = r_0, r_1, ..., r_{N/2}, i_{N/2-1}, ..., i_1    (r_k = Re X_k, i_k = Im X_k; N is even)
 * i.e. hc[k] = Re X_k for k <= N/2 and hc[N-k] = Im X_k for 0 < k < N/2 (numpy: X = rfft(x),
 * hc = concatenate([X.real[:N/2+1], X.imag[N/2-1:0:-1]]); scipy.fftpack.rfft interleaves the parts and is another format).
 * Inverse (HC2R) is the unnormalised inverse: HC2R(R2HC(x)) = N x. */
/* DFFT_DCT1 / DFFT_DST1 (not in the reference; FFTW's REDFT00 / RODFT00, scipy.fft.dct / dst with type=1, norm=None): the
 * type-I transforms of vertex-centred grids (the boundary nodes are grid points) and of Chebyshev-Gauss-Lobatto axes
 * (x_j = cos(pi j / N), j = 0..N, whose Chebyshev transform is a DCT-I of N + 1 points).  Kinds only, like DFFT_R2HC: for
 * dfft_plan_create_r2r and dfft_fft1d_r2r; dfft_plan_create* return DFFT_ERR_INVALID for transforms 16 and 17.  With N a
 * power of two:
 *   DCT-I, L = N + 1 points, N in [2, 8192]:  y_k = x_0 + (-1)^k x_N + 2 sum_{n=1}^{N-1} x_n cos(pi n k / N)
 *   DST-I, L = N - 1 points, N in [4, 8192]:  y_k = 2 sum_{n=0}^{N-2} x_n sin(pi (n+1)(k+1) / N)
 * so an axis takes L = 3, 5, 9, ..., 8193 (DCT-I) or 3, 7, 15, ..., 8191 (DST-I); any other length DFFT_ERR_UNSUPPORTED.
 * Each is its own inverse up to 2N: forward and inverse execs run the same transform on such an axis. */
enum { DFFT_DCT1 = 16, DFFT_DST1 = 17 };
/* DFFT_DCT4 / DFFT_DST4 (not in the reference; FFTW's REDFT11 / RODFT11, scipy.fft.dct / dst with type=4, norm=None): the
 * type-IV transforms of cell-centred axes whose two walls differ, N points, N a power of two in [4, 8192] (other lengths,
 * N = 2 included: DFFT_ERR_UNSUPPORTED):
 *   DCT-IV:  y_k = 2 sum_{n<N} x_n cos(pi (2n+1)(2k+1) / 4N)   Neumann at the low face (u_{-1} = u_0), Dirichlet at the high
 *                                                             one (u_N = -u_{N-1})
 *   DST-IV:  y_k = 2 sum_{n<N} x_n sin(pi (2n+1)(2k+1) / 4N)   Dirichlet at the low face, Neumann at the high one
 * Each diagonalises the 3-point second difference with those ghost rules, eigenvalues -4 sin^2(pi (2k+1) / 4N) (none zero).
 * Kinds only, like DFFT_DCT1 / DFFT_DST1: for dfft_plan_create_r2r and dfft_fft1d_r2r; dfft_plan_create* return
 * DFFT_ERR_INVALID for transforms 19 and 20.  Each is its own inverse up to 2N: forward and inverse execs run the same
 * transform on such an axis. */
enum { DFFT_DCT4 = 19, DFFT_DST4 = 20 };

typedef struct dfft_comm_s* dfft_comm_t;
typedef struct dfft_plan_s* dfft_plan_t;

/* ---- communicator (replaces MPI_Comm / MPI_Comm_size / MPI_Comm_rank, src/mpicufft.cpp:42-50) ---- */
int dfft_get_unique_id(void* id /* DFFT_UNIQUE_ID_BYTES */);
/* nranks == 1: id may be NULL and NCCL is not touched. device = CUDA ordinal this rank drives. */
int dfft_comm_create(int rank, int nranks, const void* id, int device, dfft_comm_t* comm);
int dfft_comm_destroy(dfft_comm_t comm);
int dfft_comm_rank(dfft_comm_t comm);
int dfft_comm_size(dfft_comm_t comm);

/* ---- plan = constructor + initFFT (mpicufft_slab.cpp:97-233, mpicufft_pencil.cpp:63-342) ---------- */
/* p1,p2: Partition{P1,P2} (params.hpp:39-56); slab decompositions ignore them and use the communicator
 * size.  allocate != 0: the plan allocates (and owns) its device work area, like initFFT(.., true).
 * Axis lengths: C2C plans take, per axis, a power of two in [2, 8192] or any length in [3, 4096] (lengths that are not
 * powers of two run a Bluestein pass: two FFTs of the next power of two >= 2n - 1 per line, slower than a power-of-two
 * pass of similar size, and always the sequential schedule); R2C plans take powers of two in [2, 8192] (Nz in [4, 16384]).
 * Other lengths: DFFT_ERR_UNSUPPORTED. */
int dfft_plan_create(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/,
                     int precision /*dfft_prec*/, int transform /*dfft_transform*/, size_t nx, size_t ny,
                     size_t nz, size_t p1, size_t p2, int allocate, dfft_plan_t* plan);
/* Batched plans (not in the reference): every exec transforms `batch` independent fields of the geometry above.
 *   - Fields sit back to back in every caller buffer: field f of a buffer starts f times that buffer's per-field size
 *     further, the product of its layout (dfft_get_in_size / dfft_get_out_size for full transforms,
 *     dfft_get_partial_size(d) for partial ones; counted in reals on the real side of R2C / C2R).  This is a contiguous
 *     [batch][X][Y][Z] array (torch tensor [B, X, Y, Z] or [B, X, Y, Z/2+1]).  No exec reads or writes a caller buffer
 *     beyond the per-field size of its last field, so the per-field distance is never dfft_get_domain_size().
 *   - The input of every field is left intact, as for one field.
 *   - All exec, _async, partial, tune, timer and getter calls keep their signatures; the getters describe one field, and
 *     the work area is that of one field (fields run one after another through it).
 *   - dfft_plan_tune measures field 0 of the given buffers.
 *   - dfft_get_last_launch_count, the step list and the timeline cover every launch of the exec; the phase times mark
 *     the section ends of the last field.
 *   - One-rank slab C2C plans of cubic 32^3 or 64^3 fields run a batch of two or more fields as one launch; every
 *     other batched plan runs its one-field schedule once per field (multi-rank plans: each field with its own entry
 *     rendezvous).  Both are capturable under the conditions of the _async calls below.
 * batch == 1 is dfft_plan_create.  batch == 0, or a batch whose buffers would overflow size_t: DFFT_ERR_INVALID. */
int dfft_plan_create_batched(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/,
                             int precision /*dfft_prec*/, int transform /*dfft_transform*/, size_t nx, size_t ny,
                             size_t nz, size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan);
size_t dfft_get_batch(dfft_plan_t plan); /* fields per exec (1 for dfft_plan_create), 0 for a null plan */
/* In-place plans (cuFFT and FFTW offer the same): the exec writes its output over its input, so a transform needs one
 * caller buffer instead of two.  Same arguments and validation as dfft_plan_create_batched.
 *   - Every exec (plain, _async, partial) and dfft_plan_tune require out == in; another `out` returns DFFT_ERR_INVALID.
 *     The input is consumed.  dfft_plan_tune runs the transform on the buffer, so it overwrites it as well.
 *   - The buffer holds dfft_get_domain_size() bytes per field, and field f starts f * dfft_get_domain_size() bytes in, on
 *     both sides (one distance for input and output).
 *   - R2C / C2R use the padded real layout of FFTW and cuFFT in-place transforms: real rows are 2 * (Nz/2 + 1) reals apart,
 *     and the last two reals of each row (Nz is even) are padding that is neither read nor written.  The sizes
 *     the getters report stay the logical ones (Nz reals).  In torch terms: the real view of a complex [X][Y][Nz/2+1]
 *     tensor, torch.view_as_real(buf).view(X, Y, Nz + 2), of which the first Nz columns are the data.
 *   - One rank: the work area is one slot (dfft_get_work_size_device() is half that of the out-of-place plan); the
 *     caller's buffer holds the first intermediate.  Several ranks keep their work area and schedules and save the
 *     caller's second buffer.
 *   - Output scale, partial transforms, batches, dfft_plan_tune and CUDA graph capture work as for other plans.
 * Out-of-place plans are unchanged; out == in on them is not supported (it needs an in-place plan). */
int dfft_plan_create_inplace(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/,
                             int precision /*dfft_prec*/, int transform /*dfft_transform*/, size_t nx, size_t ny,
                             size_t nz, size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan);
int dfft_plan_is_inplace(dfft_plan_t plan); /* 1 for plans of dfft_plan_create_inplace, 0 otherwise (and for a null plan) */
/* Real-to-real plans with a kind per axis (FFTW's fftw_plan_r2r with one kind per dimension): kinds[0], [1], [2] are the
 * kinds of the x, y and z axis, each DFFT_DCT (Neumann), DFFT_DST (Dirichlet), DFFT_R2HC (periodic), DFFT_DCT1 /
 * DFFT_DST1 (Neumann / Dirichlet on vertex-centred or Chebyshev axes), or DFFT_DCT4 / DFFT_DST4 (cell-centred, Neumann at
 * one face and Dirichlet at the other).  Everything said of DFFT_DCT / DFFT_DST plans above holds: real [x][y][z] buffers,
 * powers of two in [2, 8192] (type-I axes: the lengths of DFFT_DCT1 / DFFT_DST1; type-IV axes: [4, 8192]; others:
 * DFFT_ERR_UNSUPPORTED), dfft_exec_r2r* (forward: DCT-II, DST-II or R2HC on each axis; inverse: DCT-III, DST-III or
 * HC2R; DCT-I, DST-I, DCT-IV and DST-IV both ways), partial d over the first d axes in z, y, x order, each with its own
 * kind, and dfft_layout with DFFT_DCT.
 * `batch` and `inplace` (!= 0) mean what they mean for dfft_plan_create_batched / dfft_plan_create_inplace.
 *   - A round trip scales by the product over the transformed axes of N (R2HC) or 2N (DCT, DST, DCT-IV / DST-IV, and
 *     DCT-I / DST-I with their N = L - 1 / L + 1).
 *   - Three DFFT_DCT (DFFT_DST) kinds make the DFFT_DCT (DFFT_DST) plan: the same steps, description and output.  Other
 *     combinations, type-I and type-IV kinds included: dfft_plan_describe reports "r2r_kinds" and, per R2R pass, "r2r"
 *     (the kind of its axis: "dct", "dst", "r2hc", "dct1", "dst1", "dct4" or "dst4").
 *   - A null kinds or a kind outside {DFFT_DCT, DFFT_DST, DFFT_R2HC, DFFT_DCT1, DFFT_DST1, DFFT_DCT4, DFFT_DST4}:
 *     DFFT_ERR_INVALID. */
int dfft_plan_create_r2r(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/, int precision /*dfft_prec*/,
                         const int kinds[3], size_t nx, size_t ny, size_t nz, size_t p1, size_t p2, size_t batch, int inplace,
                         int allocate, dfft_plan_t* plan);
/* kinds[0..2] of the x, y and z axis of a real-to-real plan (also of DFFT_DCT / DFFT_DST plans); DFFT_ERR_INVALID for
 * R2C / C2C plans. */
int dfft_plan_get_r2r_kinds(dfft_plan_t plan, int kinds[3]);
/* Padded plans (mpi4py-fft's `padding`, for the 3/2 dealiasing rule of pseudo-spectral solvers): a physical grid of
 * nx x ny x nz points and a spectrum of kx x ky x kz modes, 1 <= k <= n per axis.  The spectral side of the plan is that of
 * an ordinary kx x ky x kz plan on the same ranks, the physical side that of the nx x ny x nz plan.
 *   - C2C axis: spectral index m in [0, K) is frequency numpy.fft.fftfreq(K)[m] * K, at position m (m < ceil(K/2)) or
 *     m + N - K of the N-point line.  R2C z axis: the modes k = 0 .. Kz/2, a spectral z extent of Kz/2 + 1.
 *   - Forward: the N-point transform, then only the kept modes are stored.  Inverse: the unnormalised inverse of the
 *     zero-embedded spectrum; the missing modes are never read.  inverse(forward(x)) = Nx*Ny*Nz times the low-pass
 *     projection of x, forward(inverse(X)) = Nx*Ny*Nz*X.
 *   - Partial d: each axis is truncated (padded) by the pass that transforms it, so the layout after d stages has K on
 *     the first d axes in z, y, x order.  The getters, batch distances and dfft_get_work_size_device follow.
 *   - Batch, output scale, Peer2Peer / All2All, dfft_plan_describe ("spectral", and "keep" on every pass with a hole) and
 *     graph capture work as for other plans; padded plans run the sequential schedule (dfft_plan_tune has no alternative).
 *   - kx = nx, ky = ny, kz = nz makes the plan of dfft_plan_create_batched: the same steps, description and output.
 *   - DFFT_DCT / DFFT_DST, or K < N on an axis whose length is not a power of two: DFFT_ERR_UNSUPPORTED.  A K of 0 or
 *     above N, transform 4, or a spectral split that leaves a rank without data: DFFT_ERR_INVALID.
 *   - No in-place form; dfft_plan_set_transform_axes other than {1, 1, 1} on a plan with some K < N: DFFT_ERR_UNSUPPORTED. */
int dfft_plan_create_padded(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/, int precision /*dfft_prec*/,
                            int transform /*dfft_transform*/, size_t nx, size_t ny, size_t nz, size_t kx, size_t ky, size_t kz,
                            size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan);
/* k[0..2] = kx, ky, kz of a padded plan; nx, ny, nz for every other plan. */
int dfft_plan_get_spectral_size(dfft_plan_t plan, size_t k[3]);
/* Pruned plans (PFFT's pruned FFTs, the doubled grid of Hockney-Eastwood free-space solvers): a transform grid of
 * nx x ny x nz points whose physical field holds data = (mx, my, mz) points, 1 <= m <= n per axis, at line positions
 * [0, m) of each axis; everything from m to n - 1 is zero and is never stored in a caller buffer.  spectral = (kx, ky, kz)
 * means what it means for dfft_plan_create_padded.  Either pointer may be NULL, which means (nx, ny, nz).
 *   - Forward: the n-point transform of the zero-embedded field; only the kept spectral modes are stored.  Inverse: the
 *     unnormalised inverse of the (zero-embedded) spectrum; only positions [0, m) of each axis are stored.
 *   - The physical side of every exec (the forward input, the inverse output) is an m-block [x_i][my][mz] (R2C / C2R:
 *     mz reals per row).  The physical x split (pencil: also the y split) is made over mx (my), not nx, so that every
 *     rank holds data.  The layout after d stages has K on the first d axes in z, y, x order and m on the others; the
 *     getters, dfft_get_domain_size, dfft_get_work_size_device and batch distances follow.
 *   - Batch, output scale, partial d, Peer2Peer / All2All, the timer and graph capture of one-rank _async execs work as
 *     for other plans.  Plans with some m < n run the sequential schedule (dfft_plan_tune has no alternative).
 *     dfft_plan_describe reports "data": [mx, my, mz] and "data": m on every pass whose physical side holds m < n points.
 *   - data = (nx, ny, nz) or NULL makes the plan of dfft_plan_create_padded with the same spectral (of
 *     dfft_plan_create_batched when both are full): the same steps, description and output.
 *   - An m of 0 or above n, a data split that leaves a rank without data, transform 4, or the spectral arguments that
 *     dfft_plan_create_padded rejects: DFFT_ERR_INVALID.  DFFT_DCT / DFFT_DST, m < n on an axis whose length is not a power
 *     of two, or an odd mz on R2C / C2R: DFFT_ERR_UNSUPPORTED.
 *   - No in-place, boxed or interleaved form; dfft_plan_set_transform_axes other than {1, 1, 1} and
 *     dfft_plan_set_strides on a plan with some m < n: DFFT_ERR_UNSUPPORTED. */
int dfft_plan_create_pruned(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/, int precision /*dfft_prec*/,
                            int transform /*dfft_transform*/, size_t nx, size_t ny, size_t nz, const size_t data[3],
                            const size_t spectral[3], size_t p1, size_t p2, size_t batch, int allocate, dfft_plan_t* plan);
/* m[0..2] = mx, my, mz of a pruned plan; nx, ny, nz for every other plan. */
int dfft_plan_get_data_size(dfft_plan_t plan, size_t m[3]);
/* Distributed 1D complex transforms (FFTW-MPI's fftw_mpi_plan_dft_1d with FFTW_MPI_SCRAMBLED_OUT / _IN): one signal of
 * n = N1 * N2 * N3 points, split over the ranks in contiguous chunks.
 *   - The signal x[n] is the grid [N1][N2][N3], n = n1 N2 N3 + n2 N3 + n3, and the plan's geometry is the
 *     DFFT_SLAB_ZY_THEN_X plan of that grid: dfft_get_in_size / _start and dfft_get_out_size / _start both give this rank's
 *     x-slab [in_size[0]][N2][N3].  This rank's chunk of the signal starts at point in_start[0] * N2 * N3.
 *   - Forward (dfft_exec_c2c, _async): out[k1][k2][k3] = X[k1 + N1 k2 + N1 N2 k3], X[k] = sum_n x[n] exp(-2 pi i n k / n):
 *     the scrambled order.  Frequency k sits at position [k % N1][(k / N1) % N2][k / (N1 N2)].  Inverse: takes that
 *     scrambled array and returns the natural-order signal, unnormalised: inverse(forward(x)) = n x.
 *   - factors: N1, N2, N3, each a power of two in [2, 8192], with N1 and N2 at least the rank count; NULL lets the
 *     library pick them: log2 n split into three parts in [1, 13], N1 and N2 >= the rank count, as balanced as possible,
 *     of equally balanced splits the one with the largest N1, then the largest N2.  dfft_plan_get_1d_factors reports them.
 *   - C2C only, DFFT_F64 or DFFT_F32, out of place, batch 1, Peer2Peer or All2All, the sequential schedule
 *     (dfft_plan_tune reports "1D plans").  dfft_plan_set_scale works as for every plan.  dfft_plan_describe reports
 *     "signal": n and "twiddle": "y" / "z" on the twiddled passes.
 *   - n not a power of two in [8, 2^39], a factor outside [2, 8192], or no default split: DFFT_ERR_UNSUPPORTED; factors
 *     whose product is not n, or N1 or N2 below the rank count: DFFT_ERR_INVALID.  DFFT_F16 / DFFT_BF16,
 *     dfft_plan_set_transform_axes other than {1, 1, 1}, dfft_plan_set_strides, dfft_plan_set_weights and partial execs
 *     (d < 3, also for dfft_plan_describe): DFFT_ERR_UNSUPPORTED. */
int dfft_plan_create_1d(dfft_comm_t comm, const dfft_config* config, int precision /*dfft_prec*/, size_t n, const size_t factors[3],
                        dfft_plan_t* plan);
/* Distributed 1D complex transforms with natural-order output (FFTW-MPI's default for fftw_mpi_plan_dft_1d): the plan
 * of dfft_plan_create_1d, with the same signal, input chunk, factors rule, precisions and refusals, and these differences.
 *   - Forward output in natural order.  With (oz_r, z0_r) rank r's part of the split of N3 over the P ranks
 *     (dfft_partition(N3, P)), rank r's out holds X[k] for k in [z0_r N1 N2, (z0_r + oz_r) N1 N2), dense, k increasing: the
 *     block [oz_r][N2][N1] of the grid [N3][N2][N1], k1 contiguous.  dfft_get_out_size gives {oz_r, N2, N1} and
 *     dfft_get_out_start {z0_r, 0, 0}, as do dfft_get_partial_size / _start for d = 3; dfft_get_domain_size covers the
 *     larger of the in and the out chunk.
 *   - Inverse: takes that natural-order chunk and returns the natural signal on the x-slabs, unnormalised:
 *     inverse(forward(x)) = n x.
 *   - Factors: N3 must also be at least the rank count (DFFT_ERR_INVALID otherwise); the default split meets that too.
 *   - dfft_plan_describe adds "order": "natural" to the plan and "transposed" to the z pass, which reads the rows of the
 *     x-slabs and stores with k1 contiguous.  On more than one rank each direction adds one exchange and one local copy
 *     (the "landing copy" forward, the "scatter copy" inverse) to the schedule of dfft_plan_create_1d. */
int dfft_plan_create_1d_natural(dfft_comm_t comm, const dfft_config* config, int precision /*dfft_prec*/, size_t n, const size_t factors[3],
                                dfft_plan_t* plan);
/* f[0..2] = N1, N2, N3 of a 1D plan (either order); DFFT_ERR_INVALID for other plans. */
int dfft_plan_get_1d_factors(dfft_plan_t plan, size_t f[3]);
/* Interleaved multi-component plans (FFTW-MPI's `howmany`): every grid point holds `components` consecutive values,
 * and each component is transformed on its own.
 *   - Every caller layout is that of the components = 1 plan with each element widened to C = components consecutive
 *     values: input [in_size[0]][in_size[1]][in_size[2]][C], output [out_size[0]][out_size[1]][out_size[2]][C], partial d
 *     likewise (torch tensors [X, Y, Z, C], with a batch [B, X, Y, Z, C]).  Component c of the output is the
 *     components = 1 transform of component c of the input.
 *   - The getters and dfft_layout describe the 3-D extents of one component; dfft_get_domain_size and
 *     dfft_get_work_size_device count all C.  `batch` fields of C components each sit back to back.
 *   - components = 1 makes the plan of dfft_plan_create_batched: the same steps, description and output.
 *   - Peer2Peer / All2All, every decomposition, partial d, uneven splits, batches, the output scale, graph capture of
 *     one-rank _async execs, the timer and dfft_debug_run_step work as for other plans.  C > 1 plans run the sequential
 *     schedule (dfft_plan_tune has one candidate); dfft_plan_describe adds "components" and lists the C2C z pass as
 *     kind 8, a TILED view mapping with b = the component, and the R2C / C2R z pass as kind 9 / 10, Nz-point lines whose
 *     real side is counted in reals.
 *   - C2C and R2C / C2R.  R2C / C2R pair components c, c + 1 as one complex Nz-point line in the z pass, so their
 *     output matches the batched plan's within rounding; C2C output equals it bit for bit.
 *   - components = 0, or a batch x components whose buffers overflow size_t: DFFT_ERR_INVALID; components > 64:
 *     DFFT_ERR_UNSUPPORTED.  With components > 1, R2R transforms, a z length that is not a power of two, an R2C / C2R Nz
 *     of 16384 (the paired z pass runs Nz-point lines) and dfft_plan_set_transform_axes other than {1, 1, 1}:
 *     DFFT_ERR_UNSUPPORTED.  No in-place or padded form. */
int dfft_plan_create_interleaved(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/, int precision /*dfft_prec*/,
                                 int transform /*dfft_transform*/, size_t nx, size_t ny, size_t nz, size_t p1, size_t p2,
                                 size_t components, size_t batch, int allocate, dfft_plan_t* plan);
size_t dfft_get_components(dfft_plan_t plan); /* 1 for every other plan, 0 for a null plan */
/* Box-distributed plans (heFFTe's box3d in and out, cuFFTMp's cufftXtSetDistribution): each rank's input and output is a
 * box of the grid the caller chooses, e.g. the Px x Py x Pz bricks of a particle-mesh or PSATD code, and the exec
 * redistributes between those boxes and the plan's own layouts on the GPU.
 *   - in_boxes / out_boxes: 6 * P values each, for rank r lo[3], hi[3] (x, y, z; half-open) at 6 r, the same arrays on every
 *     rank.  in_boxes tile the physical grid Nx x Ny x Nz, out_boxes the output grid Nx x Ny x Nzc (Nzc = Nz/2 + 1 for R2C,
 *     Nz otherwise).  NULL: that side keeps the natural layout (dfft_layout).  Boxes equal to the natural layout (and any
 *     box of one rank, which is the whole grid) make the plan of dfft_plan_create_batched: the same steps and output.
 *   - Each rank's caller buffer on a boxed side is its box as a dense [hx-lx][hy-ly][hz-lz] array, z contiguous (reals on
 *     the real side of R2C / C2R and for DCT / DST); `batch` fields sit back to back, one box volume apart.
 *   - in_boxes apply to the physical side of every exec (partial d included), out_boxes to the output of d = 3; the
 *     spectral side of d < 3 keeps its natural layout.  dfft_get_in_* report this rank's input box, dfft_get_out_* and
 *     dfft_get_partial_*(3) its output box; dfft_get_domain_size and dfft_get_work_size_device cover the box arrays.
 *   - The exec copies the boxes into the plan's layout before the first pass and out of it after the last one: with
 *     comm_method Peer2Peer each rank pushes its pieces into the owners' work areas (input) or gathers them from there
 *     (output) over peer memory, with All2All through an NCCL all-to-all.  One copy sweep per boxed side and a rendezvous
 *     or all-to-all; the FFT passes are those of the natural plan.  dfft_plan_describe reports "in_boxes" / "out_boxes"
 *     and labels the copies "reshape in" / "reshape out".
 *   - C2C (Bluestein lengths included), R2C / C2R, DCT and DST on every decomposition; batches, dfft_plan_set_scale,
 *     dfft_plan_set_transform_axes and the timer work as for other plans.  Plans with a box other than the natural one
 *     run the sequential schedule (dfft_plan_tune has one candidate).
 *   - DFFT_ERR_INVALID: another transform, a box that is empty or reaches outside its grid, overlapping boxes, or boxes
 *     that do not cover the grid.  DFFT_ERR_UNSUPPORTED: an odd z bound in the in_boxes of an R2C / C2R plan (its real
 *     rows move as pairs of reals).  No in-place, padded, interleaved or per-axis R2R form. */
int dfft_plan_create_boxes(dfft_comm_t comm, const dfft_config* config, int decomp /*dfft_decomp*/, int precision /*dfft_prec*/,
                           int transform /*dfft_transform*/, size_t nx, size_t ny, size_t nz, size_t p1, size_t p2,
                           const size_t* in_boxes, const size_t* out_boxes, size_t batch, int allocate, dfft_plan_t* plan);
int dfft_plan_destroy(dfft_plan_t plan);
/* setWorkArea(device, host) — mpicufft_slab.cpp:236-281. device must hold dfft_get_work_size_device()
 * bytes; with comm_method Peer2Peer and more than one rank it must be the base of a cudaMalloc
 * allocation (it is exported to the peers with CUDA IPC).  host is accepted and unused. */
int dfft_set_work_area(dfft_plan_t plan, void* device, void* host);

/* ---- execute (mpicufft_slab.cpp:771-871, mpicufft_pencil.cpp:1643-1839) ----------------------------
 * Collective over the communicator, unnormalised in both directions (inverse(forward(x)) = Nx*Ny*Nz*x).
 * Layouts, z contiguous:
 *   real/complex input  [in_size[0]][in_size[1]][in_size[2]]     (dfft_get_in_size)
 *   complex output      [out_size[0]][out_size[1]][out_size[2]]  (dfft_get_out_size)
 * `out` of exec_r2c / `in` of exec_c2r must hold dfft_get_domain_size() bytes.
 * out == in needs a plan of dfft_plan_create_inplace (see there); other plans take two distinct buffers.
 * The plain calls return after the device has finished (the reference's cudaDeviceSynchronize);
 * the _async calls enqueue on `stream` (a cudaStream_t) and return. */
int dfft_exec_r2c(dfft_plan_t plan, void* out, const void* in);
int dfft_exec_c2r(dfft_plan_t plan, void* out, const void* in);
/* direction: -1 forward (DFFT_FORWARD), +1 inverse; plan must be DFFT_C2C. */
#define DFFT_FORWARD (-1)
#define DFFT_INVERSE (1)
int dfft_exec_c2c(dfft_plan_t plan, void* out, const void* in, int direction);
/* Real-to-real plans: direction DFFT_FORWARD runs DCT-II / DST-II / R2HC, DFFT_INVERSE DCT-III / DST-III / HC2R. */
int dfft_exec_r2r(dfft_plan_t plan, void* out, const void* in, int direction);
/* pencil execR2C(out,in,d)/execC2R(out,in,d): transform only the first d dimensions (z; z,y; z,y,x). */
int dfft_exec_r2c_partial(dfft_plan_t plan, void* out, const void* in, int d);
int dfft_exec_c2r_partial(dfft_plan_t plan, void* out, const void* in, int d);
int dfft_exec_c2c_partial(dfft_plan_t plan, void* out, const void* in, int direction, int d);
int dfft_exec_r2r_partial(dfft_plan_t plan, void* out, const void* in, int direction, int d);

/* CUDA graphs: an _async call on a stream that is being captured (cudaStreamBeginCapture, torch.cuda.graph) records
 * the transform's kernels into the graph instead of running them, for plans of one rank:
 *   - the same direction must have run eagerly on this plan first (the first exec sets up tables and kernel
 *     attributes, which a capture cannot do); otherwise DFFT_ERR_STATE and nothing is captured;
 *   - multi-rank plans return DFFT_ERR_UNSUPPORTED and capture nothing;
 *   - a captured exec records no timer events and leaves the launch count, the phase and step times and the stream
 *     dfft_plan_wait waits for as the last eager exec left them;
 *   - the graph replays the buffers it was captured with and stays valid until the plan is destroyed, re-tuned
 *     (dfft_plan_tune) or given a new work area (dfft_set_work_area);
 *   - execs of one plan, eager or replayed, must be ordered on the device with respect to each other (one stream, or
 *     events), as for eager execs alone.
 * The plain synchronous calls and dfft_plan_tune cannot be captured. */
int dfft_exec_r2c_async(dfft_plan_t plan, void* out, const void* in, void* stream);
int dfft_exec_c2r_async(dfft_plan_t plan, void* out, const void* in, void* stream);
int dfft_exec_c2c_async(dfft_plan_t plan, void* out, const void* in, int direction, void* stream);
int dfft_exec_r2r_async(dfft_plan_t plan, void* out, const void* in, int direction, void* stream);
/* Output scale (not in the reference; cuFFT has none either).  Every exec of a direction multiplies each output value by
 * that direction's scale: the real and imaginary parts of complex outputs, the real values of C2R outputs.  It applies to
 * the plain and _async calls, R2C / C2R / C2C, partial transforms (the value is used as given), every field of a batched
 * plan, and every decomposition.  The kernel that stores the final values multiplies them, in the plan's precision, as
 * they leave the registers: no extra launch and no extra memory traffic.  The result equals the unscaled output times the
 * scale computed in the same precision, bit for bit (f32 plans round the scale to float once).  Defaults (1, 1): the plan
 * runs exactly its unscaled kernels.
 * Normalisations, with N the product of the transformed lengths (Nx*Ny*Nz, or that of the first d for partial ones):
 *   backward (torch / numpy default, cuFFT round trips)  (1, 1/N)
 *   ortho                                                (1/sqrt(N), 1/sqrt(N))
 *   forward                                              (1/N, 1)
 * Local to the calling rank, not collective: set the same values on every rank of a multi-rank plan.  A null plan, or a
 * NaN or infinite scale, returns DFFT_ERR_INVALID.  A CUDA graph replays the scale in effect when it was captured.
 * dfft_plan_set_scale (even to the values already set) makes every direction run eagerly once more before it can be
 * captured again (DFFT_ERR_STATE otherwise), as for the first exec. */
int dfft_plan_set_scale(dfft_plan_t plan, double forward_scale, double inverse_scale);
/* Either pointer may be NULL. */
int dfft_plan_get_scale(dfft_plan_t plan, double* forward_scale, double* inverse_scale);
/* Per-axis spectral weights (not in the reference; cuFFT offers this through load and store callbacks only).  Every exec
 * multiplies the spectrum by the separable table W[kx,ky,kz] = wx[kx] * wy[ky] * wz[kz]: derivatives (i k), half-cell
 * shifts (exp(-+i pi k / N)) and separable filters without an extra sweep over the spectrum.
 *   - weights[0], [1], [2] belong to the x, y and z axis, the order of dfft_plan_create_r2r's kinds.  Each is NULL (all
 *     ones) or a device pointer on the plan's device to complex values of the plan's precision (double2 for DFFT_F64,
 *     float2 for DFFT_F32), as many as the axis's spectral extent: Kx, Ky, Kz for C2C, Kz / 2 + 1 on z for R2C / C2R (K = N
 *     without padding).  Entry m belongs to spectral position m as the caller stores it: numpy's fftfreq order for C2C,
 *     the K stored positions of padded and pruned plans.
 *   - Forward: out = W * F(x).  Inverse: out = F^-1(W * X).  Both unnormalised, then times the direction's output scale
 *     (dfft_plan_set_scale).  Partial d: the weights of the first d axes in z, y, x order; kept axes
 *     (dfft_plan_set_transform_axes) ignore theirs.  C2R transforms the stored half spectrum times W: for a real result to
 *     mean anything W must be Hermitian, e.g. i k with its Nyquist entry zeroed.
 *   - The pass that transforms an axis multiplies its spectral side as the values pass through the registers: forward as
 *     it stores, inverse as it loads.  No extra launch and no extra memory traffic beyond one table read per value.
 *   - The caller owns the arrays.  The plan keeps the pointers, not copies: every exec reads the current contents, which
 *     may change between execs in stream order like an input buffer.
 *   - The first call must come before the plan builds a schedule (its first exec, dfft_plan_tune or dfft_plan_describe),
 *     DFFT_ERR_STATE otherwise; it makes the plan a weighted plan, which runs the sequential schedule (no fused z + y stage,
 *     batched stage or overlapped schedule).  Later calls may re-point any axis, or set it to NULL, at any time.
 *   - Local to the calling rank: every rank of a multi-rank plan makes the first call or none does, each with its own
 *     pointers to the same values.  Geometry-only plans accept any pointer value and never dereference it.
 *   - A CUDA graph keeps the pointers in effect when it was captured and reads their contents at replay.  A call makes
 *     every direction run eagerly once more before it can be captured again (DFFT_ERR_STATE otherwise).
 *   - DFFT_ERR_INVALID: a null plan or array, or a pointer not aligned to its element.  DFFT_ERR_UNSUPPORTED: interleaved
 *     plans of more than one component, real-to-real plans (DCT / DST and per-axis kinds) and 16-bit plans. */
int dfft_plan_set_weights(dfft_plan_t plan, const void* const weights[3]);
/* The pointers set last, NULL where none was set. */
int dfft_plan_get_weights(dfft_plan_t plan, const void* weights[3]);
/* Untransformed axes (not in the reference; FFTW's guru "howmany" dimensions, 2DECOMP&FFT's standalone transposes).
 * transform[0], [1], [2] belong to the x, y and z axis, the order of dfft_plan_create_r2r's kinds: 1 transforms that axis,
 * 0 keeps it.  A kept axis is redistributed exactly as a transformed one would be, but its values are not transformed: an
 * exec with x kept transforms z and y and delivers the output distribution (x whole on every rank), the layout a
 * tridiagonal or banded solve along x needs.  All three kept: a distributed transpose.  Default {1, 1, 1}.
 *   - Layouts, getters, dfft_get_domain_size and work sizes do not change.  A kept axis still needs a length its plan's
 *     transform accepts.  R2R kinds of kept axes are ignored (dfft_plan_get_r2r_kinds still reports them).
 *   - Partial d keeps its meaning: the first d stages in z, y, x order, each transformed or kept.  A round trip scales by
 *     the product over the transformed axes among them of N (C2C, R2C, R2HC) or 2N (DCT, DST).
 *   - A kept axis is one copy pass where a transform would run, none where the copy would only move memory on one rank
 *     (DESIGN.md section 3.12).  These plans run the sequential schedule (dfft_plan_tune has one candidate).  Scale,
 *     batches, in-place plans, every decomposition, Peer2Peer and All2All and graph capture work as for other plans.
 *   - dfft_plan_describe: copy steps have kind 6 (contiguous) or 7 (strided) and "n"; plans with a kept axis report
 *     "transform_axes".
 * A null plan or array, an entry that is not 0 or 1, or an R2C / C2R plan with z kept: DFFT_ERR_INVALID.  Once the plan
 * has built a schedule (its first exec, dfft_plan_tune or dfft_plan_describe): DFFT_ERR_STATE — set it once, right after
 * creation.  Local to the calling rank: set the same values on every rank. */
int dfft_plan_set_transform_axes(dfft_plan_t plan, const int transform[3]);
int dfft_plan_get_transform_axes(dfft_plan_t plan, int transform[3]);
/* Embedded layouts (not in the reference; cuFFT's inembed / istride / idist, FFTW's advanced interface): each rank's block
 * of a side is read or written inside a larger caller array, e.g. the interior of a field with ghost cells or a torch
 * slice A[h:-h, h:-h, h:-h], with no pack or unpack around the exec.
 *   - in_strides / out_strides: {field, x, y} strides of that side's caller array, in its elements (complex values on
 *     complex sides; reals on the real side of R2C / C2R and on every side of R2R plans); z is contiguous.  NULL keeps that
 *     side dense.  The caller passes a pointer to the block's first element, as torch's data_ptr() of a slice is.
 *   - `in` is the physical side: the forward input and the inverse output, partial d included.  `out` is the output of
 *     d = 3 (the forward output, the inverse input); the spectral side of a partial exec stays dense, as for boxes.
 *   - The block is this rank's dfft_get_in_size / dfft_get_out_size (its box on box plans).  Strides must keep its points
 *     apart: y >= the block's z extent, x >= ny * y, field >= nx * x, and every stride even on the real side of R2C / C2R
 *     (its rows move as pairs of reals); otherwise DFFT_ERR_INVALID.  At exec, a pointer on an embedded side that is not
 *     aligned to its element (a pair of reals on the real side of R2C / C2R) returns DFFT_ERR_INVALID.
 *   - The FFT passes read and write the caller's array through the strides: the first pass reads it, the last one writes
 *     it, and no element outside the block is touched.  Such plans run the sequential schedule (no overlapped schedule,
 *     fused z + y stage or one-launch batched stage; dfft_plan_tune has one candidate).  Every rank calls this, or none
 *     does; each with its own values, since the caller's buffers are local.
 *   - C2C (Bluestein lengths included), R2C / C2R and every R2R kind on every decomposition, with batches, scale, partial
 *     d, kept axes, padded plans and box plans (the box is the block).  dfft_plan_describe reports "in_strides" /
 *     "out_strides".  In-place and interleaved plans: DFFT_ERR_UNSUPPORTED.  Once the plan has built a schedule:
 *     DFFT_ERR_STATE, as for dfft_plan_set_transform_axes.
 * dfft_plan_get_strides reports the strides of each side, those of the dense block for a side without them; either
 * pointer may be NULL. */
int dfft_plan_set_strides(dfft_plan_t plan, const long long in_strides[3], const long long out_strides[3]);
int dfft_plan_get_strides(dfft_plan_t plan, long long in_strides[3], long long out_strides[3]);
/* Waits for the stream of the last eager _async call and reports a device-side failure (rendezvous or fused-stage
 * timeout), if any.  After replaying a graph, synchronise the replay stream first; dfft_plan_wait then reports the
 * errors the replayed kernels recorded. */
int dfft_plan_wait(dfft_plan_t plan);

/* ---- getters (mpicufft.hpp:65-78, mpicufft_slab.hpp:122-125, mpicufft_pencil.hpp:112-122) ---------- */
int dfft_get_in_size(dfft_plan_t plan, size_t size[3]);
int dfft_get_in_start(dfft_plan_t plan, size_t start[3]);
int dfft_get_out_size(dfft_plan_t plan, size_t size[3]);
int dfft_get_out_start(dfft_plan_t plan, size_t start[3]);
/* layout after d transformed dimensions (pencil partial transforms); d = 3 equals get_out_*. */
int dfft_get_partial_size(dfft_plan_t plan, int d, size_t size[3]);
int dfft_get_partial_start(dfft_plan_t plan, int d, size_t start[3]);
size_t dfft_get_domain_size(dfft_plan_t plan);      /* bytes, getDomainSize() */
size_t dfft_get_work_size_device(dfft_plan_t plan); /* bytes, getWorkSizeDevice() */
size_t dfft_get_work_size_host(dfft_plan_t plan);   /* always 0: nothing is staged through the host */
void* dfft_get_work_area_device(dfft_plan_t plan);
int dfft_get_rank(dfft_plan_t plan);
int dfft_get_world_size(dfft_plan_t plan);

/* ---- partition arithmetic without a GPU (initFFT's split rule, mpicufft_slab.cpp:112-128,
 *      mpicufft_pencil.cpp:89-110): sizes[p] = n/parts + (p < n%parts), starts = prefix sums. -------- */
int dfft_partition(size_t n, size_t parts, size_t* sizes, size_t* starts);
/* Geometry of any rank of a would-be plan, no device needed (used by the CPU tests and by callers that
 * size their buffers before creating the plan).  which: 0 in, 1 after d=1, 2 after d=2, 3 out. */
int dfft_layout(int decomp, int transform, size_t nx, size_t ny, size_t nz, size_t p1, size_t p2,
                int rank, int which, size_t size[3], size_t start[3]);

/* ---- plan-time measurement ---------------------------------------------------------------------------------
 * The reference offers Sync and Streams variants of every transposition and leaves the choice to the user's own
 * benchmark sweeps (jobs/ ** /benchmarks_base.json).  dfft_plan_tune makes it once, at plan time, like FFTW_MEASURE:
 * it runs the transform on the caller's buffers with the sequential schedule and with overlapped schedules that give the
 * exchanging pass different numbers of CTAs, and keeps the fastest (slowest rank decides).  Collective; `out` is
 * overwritten, `in` is not — except on in-place plans, where out == in and the buffer is overwritten.  Only plans with
 * send_method Streams have alternatives.  Returns the candidate index.
 * Not capturable: call it before capturing, never on a capturing stream. */
int dfft_plan_tune(dfft_plan_t plan, void* out, const void* in, int inverse, int reps);
const char* dfft_plan_tune_report(dfft_plan_t plan);

/* ---- phase timer (include/timer.hpp, src/timer.cpp; section names mpicufft_slab.hpp:209-223,
 *      mpicufft_pencil.hpp:263-287) -------------------------------------------------------------------
 * Cumulative milliseconds since the start of the last exec, measured with CUDA events. */
int dfft_timer_enable(dfft_plan_t plan, int enable);
int dfft_get_phase_count(dfft_plan_t plan);
const char* dfft_get_phase_name(dfft_plan_t plan, int i);
int dfft_get_phase_times(dfft_plan_t plan, double* ms, int capacity);
/* Per-step GPU time of the last timed exec, in launch order: one entry per FFT pass / rendezvous / all-to-all
 * (labels such as "z pass", "y pass", "x pass", "rendezvous 2", "nccl all-to-all"). */
int dfft_get_step_count(dfft_plan_t plan);
const char* dfft_get_step_label(dfft_plan_t plan, int i);
int dfft_get_step_times(dfft_plan_t plan, double* ms, int capacity);
/* Timeline of the last timed exec (also for overlapped schedules, whose steps run on three streams): step i ran on
 * plan stream stream[i] (0 the caller's, 1 exchange, 2 follow-up) from begin_ms[i] to end_ms[i] after the exec's start.
 * Returns the number of steps. */
int dfft_get_timeline(dfft_plan_t plan, double* begin_ms, double* end_ms, int* stream, int capacity);
const char* dfft_get_timeline_label(dfft_plan_t plan, int i);
/* Collective: gathers the section times of the last timed exec to rank 0, which appends one block to the CSV
 * in the reference's schema (src/timer.cpp:58-101).  Called automatically after every non-warm-up
 * synchronous exec when Configurations::benchmark_dir is set. */
int dfft_timer_gather(dfft_plan_t plan);
const char* dfft_timer_csv_path(dfft_plan_t plan);
/* GPU time of the local FFT passes and of the exchange steps of the last timed exec (ms). */
int dfft_get_last_breakdown(dfft_plan_t plan, double* fft_ms, double* exchange_ms, double* total_ms);

/* number of kernels the last exec launched (FFT passes + rendezvous kernels; NCCL's own not counted) */
int dfft_get_last_launch_count(dfft_plan_t plan);

const char* dfft_last_error_string(void);
int dfft_version(void);

/* ---- single-axis building block (what one cufftExec* of the reference's plans computes) ------------
 * Batched 1D transform of `lines` contiguous lines of length n on the current device.
 * kind: 0 C2C, 1 R2C (n real -> n/2+1 complex), 2 C2R.  Exposed for tests and micro-benchmarks.
 * Lengths: C2C (kind 0, dfft_fft1d_strided, dfft_fft1d_general) a power of two in [2, 8192] or any length in [3, 4096];
 * R2C / C2R powers of two only.  Other lengths: DFFT_ERR_UNSUPPORTED.  out == in is allowed. */
int dfft_fft1d_contig(int precision, int kind, int direction, size_t n, size_t lines, void* out,
                      size_t out_pitch, const void* in, size_t in_pitch, void* stream);
/* Batched 1D C2C along the middle axis of a [a][n][b] array (b contiguous). */
int dfft_fft1d_strided(int precision, int direction, size_t a, size_t n, size_t b, void* out, const void* in,
                       void* stream);

/* DCT / DST / R2HC (transform DFFT_DCT, DFFT_DST or DFFT_R2HC; forward type II or R2HC, inverse type III or HC2R,
 * unnormalised) along the middle axis of a dense real [a][n][b] array, b contiguous; n a power of two in [2, 8192].
 * DFFT_DCT1 / DFFT_DST1: DCT-I / DST-I in both directions, n one of the lengths of that kind.  DFFT_DCT4 / DFFT_DST4:
 * DCT-IV / DST-IV in both directions, n a power of two in [4, 8192].  out == in is allowed. */
int dfft_fft1d_r2r(int precision, int transform, int direction, size_t n, size_t a, size_t b, void* out, const void* in,
                   void* stream);

/* ---- test hooks -----------------------------------------------------------------------------------------
 * Geometry-only communicator: plans created on it never touch CUDA or NCCL (slot addresses are synthetic,
 * ((rank+1) << 44) + slot * slot_bytes) and cannot execute; dfft_plan_describe returns the step list of a
 * schedule (passes with their views, rendezvous, all-to-all counts) as JSON so that the CPU tests can replay
 * the data movement of any rank count with numpy (tests/test_schedule_emulation.py). */
int dfft_comm_create_dry(int rank, int nranks, dfft_comm_t* comm);
int dfft_plan_describe(dfft_plan_t plan, int inverse, int d, char* buf, size_t capacity, size_t* needed);
/* Runs one pass step of a geometry-only plan's schedule on the current device, with the kernels and parameters an exec
 * launches for it (tables, tile choice, CTA limit, output scale), then synchronises `stream`.  With the steps of every rank
 * run in lock step and the all-to-all steps done as copies, one GPU replays a multi-rank exec
 * (tests/test_gpu_schedule_replay.py).
 *   - step indexes the schedule of (inverse, d), field the field of a per-field batched plan: item i of
 *     dfft_plan_describe's list is (field i / steps, step i % steps).
 *   - work[r] is rank r's work area of work_bytes bytes (P entries): a slot address ((r+1) << 44) + off maps to
 *     work[r] + off.  Views on the caller's buffers are offsets into in / out (in_bytes / out_bytes), as in an exec.
 *   - Every element of both views must lie inside the buffer it maps to; otherwise DFFT_ERR_INVALID and nothing runs.
 *   - Rendezvous and all-to-all steps, the fused z + y stage and the batched stage: DFFT_ERR_UNSUPPORTED.  A plan not made
 *     on dfft_comm_create_dry: DFFT_ERR_STATE. */
int dfft_debug_run_step(dfft_plan_t plan, int inverse, int d, size_t field, int step, void* const* work, size_t work_bytes,
                        void* out, size_t out_bytes, const void* in, size_t in_bytes, void* stream);

/* Batched 1D C2C along n of element (i0, i1, n, ib) at  i0*strides[0] + i1*strides[1] + n*strides[2] + ib
 * (elements; ib contiguous, extents a0 x a1 x n x b) — the general strided view the plan's passes use. */
int dfft_fft1d_general(int precision, int direction, size_t n, size_t a0, size_t a1, size_t b, void* out,
                       const long long out_strides[3], const void* in, const long long in_strides[3], void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DFFT_H_ */
