// dfft.hpp — header-only C++ shim that re-creates the reference's class and method names
// (/root/reference/include/mpicufft.hpp:55-105, mpicufft_slab.hpp:88-125, mpicufft_slab_z_then_yx.hpp,
// mpicufft_pencil.hpp:71-122, params.hpp:24-93) on top of the C ABI in dfft.h, so that caller code
// written against eggersn/DistributedFFT compiles with `MPI_Comm` replaced by `dfft_comm_t`:
//
//     Configurations config{true, 0, Peer2Peer, Sync, "", Peer2Peer, Sync};
//     MPIcuFFT_Slab<double> fft(config, comm);
//     GlobalSize gs(Nx, Ny, Nz);
//     fft.initFFT(&gs, true);
//     fft.execR2C(out_d, in_d);
//
// Error convention follows the reference: failures print the message and exit(EXIT_FAILURE)
// (/root/reference/src/slab/default/mpicufft_slab.cpp:23-29); the pencil class throws
// std::runtime_error for an uninitialised plan (/root/reference/src/pencil/mpicufft_pencil.cpp:22-25).
#pragma once
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <stdexcept>
#include <string>
#include <vector>

#include "dfft.h"

struct GlobalSize {
    GlobalSize(size_t Nx_, size_t Ny_, size_t Nz_) : Nx(Nx_), Ny(Ny_), Nz(Nz_), Nz_out(Nz_ / 2 + 1) {}
    size_t Nx, Ny, Nz, Nz_out;
};
struct Partition { size_t P1, P2; };
struct Slab_Partition : public Partition { Slab_Partition(size_t P1_) { P1 = P1_; P2 = 1; } };
struct Pencil_Partition : public Partition { Pencil_Partition(size_t P1_, size_t P2_) { P1 = P1_; P2 = P2_; } };

struct Partition_Dimensions {
    std::vector<size_t> size_x, size_y, size_z, start_x, start_y, start_z;
    // params.hpp:60-64: appends the running sums of the three size lists to the start lists
    void computeOffsets() {
        const std::vector<size_t>* sizes[3] = {&size_x, &size_y, &size_z};
        std::vector<size_t>* starts[3] = {&start_x, &start_y, &start_z};
        for (int a = 0; a < 3; ++a) {
            size_t at = 0;
            for (size_t v : *sizes[a]) { starts[a]->push_back(at); at += v; }
        }
    }
};

enum CommunicationMethod { Peer2Peer, All2All };
enum SendMethod { Sync, Streams, MPI_Type };
struct Configurations {
    bool cuda_aware;
    int warmup_rounds;
    CommunicationMethod comm_method;
    SendMethod send_method;
    std::string benchmark_dir;
    CommunicationMethod comm_method2;
    SendMethod send_method2;
};

namespace dfft_shim {
template <typename T> struct prec;
template <> struct prec<float> { static constexpr int value = DFFT_F32; };
template <> struct prec<double> { static constexpr int value = DFFT_F64; };
// 16-bit plans (DFFT_F16 / DFFT_BF16): MPIcuFFT_Slab<__half> etc. once the caller has included cuda_fp16.h / cuda_bf16.h
#ifdef __CUDA_FP16_H__
template <> struct prec<__half> { static constexpr int value = DFFT_F16; };
#endif
#ifdef __CUDA_BF16_H__
template <> struct prec<__nv_bfloat16> { static constexpr int value = DFFT_BF16; };
#endif
inline void die(int rc, const char* file, int line) {
    if (rc < 0) {
        std::printf("Error %d at %s:%d: %s\n", rc, file, line, dfft_last_error_string());
        std::exit(EXIT_FAILURE);
    }
}
}  // namespace dfft_shim
#define DFFT_CALL(x) dfft_shim::die((x), __FILE__, __LINE__)

template <typename T>
class MPIcuFFT {
public:
    MPIcuFFT(Configurations config_, dfft_comm_t comm_, int /*max_world_size*/ = -1, int transform_ = DFFT_R2C)
        : config(config_), comm(comm_), transform(transform_) {
        pidx = dfft_comm_rank(comm);
        pcnt = dfft_comm_size(comm);
    }
    // not in the reference: a real-to-real plan with a kind per axis — kinds_[0..2] of x, y, z, each DFFT_DCT, DFFT_DST,
    // DFFT_R2HC, DFFT_DCT1, DFFT_DST1, DFFT_DCT4 or DFFT_DST4; initFFT creates it with dfft_plan_create_r2r and execR2R runs it
    MPIcuFFT(Configurations config_, dfft_comm_t comm_, int max_world_size, const int (&kinds_)[3])
        : MPIcuFFT(config_, comm_, max_world_size, DFFT_R2HC) {
        per_axis = true;
        for (int a = 0; a < 3; ++a) kinds[a] = kinds_[a];
    }
    virtual ~MPIcuFFT() { if (plan) dfft_plan_destroy(plan); }

    virtual void initFFT(GlobalSize* global_size, Partition* partition, bool allocate = true) = 0;
    // not in the reference: every exec transforms `batch` fields, back to back in each buffer (dfft_plan_create_batched)
    void initFFT(GlobalSize* global_size, Partition* partition, bool allocate, size_t batch) {
        struct Reset { size_t& b; ~Reset() { b = 1; } } reset{batch_};
        batch_ = batch;
        initFFT(global_size, partition, allocate);
    }
    // not in the reference: an in-place plan (dfft_plan_create_inplace): every exec takes out == in and overwrites its
    // input; R2C / C2R use padded real rows of 2 * (Nz/2 + 1) reals
    void initFFT(GlobalSize* global_size, Partition* partition, bool allocate, size_t batch, bool inplace) {
        struct Reset { bool& i; ~Reset() { i = false; } } reset{inplace_};
        inplace_ = inplace;
        initFFT(global_size, partition, allocate, batch);
    }
    // not in the reference: a padded plan (dfft_plan_create_padded): global_size is the physical grid, spectral the
    // Kx x Ky x Kz spectrum it keeps (the forward truncates to it, the inverse zero-pads it), 1 <= K <= N per axis
    void initFFT(GlobalSize* global_size, GlobalSize* spectral, Partition* partition, bool allocate = true, size_t batch = 1) {
        struct Reset { GlobalSize*& s; ~Reset() { s = nullptr; } } reset{spectral_};
        spectral_ = spectral;
        initFFT(global_size, partition, allocate, batch);
    }
    // not in the reference: a pruned plan (dfft_plan_create_pruned): global_size is the transform grid, data the Mx x My x Mz
    // block of the field at the origin (zero beyond: the forward reads only it, the inverse stores only it), spectral the
    // spectrum it keeps (null: all of it), 1 <= M, K <= N per axis
    void initFFT(GlobalSize* global_size, GlobalSize* data, GlobalSize* spectral, Partition* partition, bool allocate = true, size_t batch = 1) {
        struct Reset { GlobalSize*& d; GlobalSize*& s; ~Reset() { d = nullptr; s = nullptr; } } reset{data_, spectral_};
        data_ = data;
        spectral_ = spectral;
        initFFT(global_size, partition, allocate, batch);
    }
    // not in the reference: an interleaved plan (dfft_plan_create_interleaved): every grid point holds `components`
    // consecutive values, each component transformed on its own ([x][y][z][C] buffers).  A named method, so that it cannot
    // be mistaken for the (batch, inplace) overload.
    void initFFTInterleaved(GlobalSize* global_size, Partition* partition, size_t components, bool allocate = true, size_t batch = 1) {
        struct Reset { size_t& c; ~Reset() { c = 1; } } reset{components_};
        components_ = components;
        initFFT(global_size, partition, allocate, batch);
    }
    size_t getComponents() const { return dfft_get_components(plan); }
    // not in the reference: a distributed 1D C2C transform of one n-point signal (dfft_plan_create_1d), the slab plan of the
    // grid factors[0..2] = N1 x N2 x N3 (null: the library's choice, getFactors).  Each rank's buffers are its x-slab of that
    // grid on both sides, its chunk of the signal from point getInStart()[0] * N2 * N3; the forward output is in scrambled
    // order, frequency k at [k % N1][(k / N1) % N2][k / (N1 N2)] (dfft.h).  The plan's class runs it with its C2C exec.
    // natural (dfft_plan_create_1d_natural): the forward output in natural order instead, each rank's out its chunk
    // [getOutSize()[0]][N2][N1] of the spectrum, frequencies from getOutStart()[0] * N1 * N2 on.
    void initFFT1d(size_t n, const size_t* factors = nullptr, bool natural = false) {
        const dfft_config c = make_config();
        if (plan) { dfft_plan_destroy(plan); plan = nullptr; }
        if (natural) DFFT_CALL(dfft_plan_create_1d_natural(comm, &c, dfft_shim::prec<T>::value, n, factors, &plan));
        else DFFT_CALL(dfft_plan_create_1d(comm, &c, dfft_shim::prec<T>::value, n, factors, &plan));
        initialized = true;
    }
    // N1, N2, N3 of a 1D plan
    void getFactors(size_t* f) const { DFFT_CALL(dfft_plan_get_1d_factors(plan, f)); }
    // not in the reference: a box plan (dfft_plan_create_boxes): in_boxes / out_boxes hold lo[3], hi[3] of every rank in
    // rank order (6 values each; null: the natural layout), and each rank's buffers are its boxes
    void initFFT(GlobalSize* global_size, Partition* partition, const size_t* in_boxes, const size_t* out_boxes, bool allocate = true,
                 size_t batch = 1) {
        struct Reset { const size_t*& i; const size_t*& o; ~Reset() { i = nullptr; o = nullptr; } } reset{in_boxes_, out_boxes_};
        in_boxes_ = in_boxes;
        out_boxes_ = out_boxes;
        initFFT(global_size, partition, allocate, batch);
    }
    // kx, ky, kz of a padded plan; Nx, Ny, Nz of every other plan
    void getSpectralSize(size_t* k) const { DFFT_CALL(dfft_plan_get_spectral_size(plan, k)); }
    // mx, my, mz of a pruned plan; Nx, Ny, Nz of every other plan
    void getDataSize(size_t* m) const { DFFT_CALL(dfft_plan_get_data_size(plan, m)); }
    size_t getBatch() const { return dfft_get_batch(plan); }
    bool isInPlace() const { return dfft_plan_is_inplace(plan) != 0; }
    // not in the reference: output scale of every forward / inverse exec (dfft_plan_set_scale; after initFFT).  For
    // normalised round trips use setScale(1, 1.0 / (Nx * Ny * Nz)).
    void setScale(double forward_scale, double inverse_scale) { DFFT_CALL(dfft_plan_set_scale(plan, forward_scale, inverse_scale)); }
    void getScale(double& forward_scale, double& inverse_scale) const { DFFT_CALL(dfft_plan_get_scale(plan, &forward_scale, &inverse_scale)); }
    // not in the reference: per-axis spectral weights (dfft_plan_set_weights; after initFFT, the first call before the
    // first exec).  Device arrays of complex T (nullptr = all ones); the plan reads them at every exec.
    void setWeights(const void* wx, const void* wy, const void* wz) {
        const void* const w[3] = {wx, wy, wz};
        DFFT_CALL(dfft_plan_set_weights(plan, w));
    }
    // not in the reference: transform (true) or keep (false) the x, y, z axis (dfft_plan_set_transform_axes; after
    // initFFT, before the first exec).  setTransformAxes(false, true, true) leaves x untransformed and whole on every rank.
    void setTransformAxes(bool x, bool y, bool z) {
        const int t[3] = {x ? 1 : 0, y ? 1 : 0, z ? 1 : 0};
        DFFT_CALL(dfft_plan_set_transform_axes(plan, t));
    }
    // not in the reference: {field, x, y} strides of the caller's arrays on the physical side (in) and the output of d = 3
    // (out), in that side's elements, z contiguous (dfft_plan_set_strides; after initFFT, before the first exec).  Null keeps
    // a side dense; the exec takes a pointer to each block's first element.
    void setStrides(const long long in[3], const long long out[3]) { DFFT_CALL(dfft_plan_set_strides(plan, in, out)); }
    virtual void setWorkArea(void* device = nullptr, void* host = nullptr) { DFFT_CALL(dfft_set_work_area(plan, device, host)); }
    virtual void execR2C(void* out, const void* in) = 0;
    // not in the reference: real-to-real transform of a plan constructed with transform_ = DFFT_DCT or DFFT_DST, or with
    // per-axis kinds (forward type II / R2HC, inverse type III / HC2R, unnormalised); d < 3 transforms only the first d
    // dimensions
    void execR2R(void* out, const void* in, int direction, int d = 3) {
        DFFT_CALL(d == 3 ? dfft_exec_r2r(plan, out, in, direction) : dfft_exec_r2r_partial(plan, out, in, direction, d));
    }

    virtual void getInSize(size_t* isize) { DFFT_CALL(dfft_get_in_size(plan, isize)); }
    virtual void getInStart(size_t* istart) { DFFT_CALL(dfft_get_in_start(plan, istart)); }
    virtual void getOutSize(size_t* osize) { DFFT_CALL(dfft_get_out_size(plan, osize)); }
    virtual void getOutStart(size_t* ostart) { DFFT_CALL(dfft_get_out_start(plan, ostart)); }

    size_t getDomainSize() const { return dfft_get_domain_size(plan); }
    size_t getWorkSizeDevice() const { return dfft_get_work_size_device(plan); }
    size_t getWorkSizeHost() const { return dfft_get_work_size_host(plan); }
    void* getWorkAreaDevice() const { return dfft_get_work_area_device(plan); }
    void* getWorkAreaHost() const { return nullptr; }
    int getRank() const { return pidx; }
    int getWorldSize() const { return pcnt; }
    dfft_plan_t handle() const { return plan; }

protected:
    dfft_config make_config() const {
        dfft_config c{};
        c.cuda_aware = config.cuda_aware; c.warmup_rounds = config.warmup_rounds;
        c.comm_method = config.comm_method; c.send_method = config.send_method;
        c.benchmark_dir = config.benchmark_dir.empty() ? nullptr : config.benchmark_dir.c_str();
        c.comm_method2 = config.comm_method2; c.send_method2 = config.send_method2;
        return c;
    }
    void create(int decomp, GlobalSize* gs, size_t p1, size_t p2, bool allocate) {
        const dfft_config c = make_config();
        if (plan) { dfft_plan_destroy(plan); plan = nullptr; }
        if (in_boxes_ || out_boxes_)
            DFFT_CALL(dfft_plan_create_boxes(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, p1, p2, in_boxes_,
                                             out_boxes_, batch_, allocate ? 1 : 0, &plan));
        else if (components_ != 1)
            DFFT_CALL(dfft_plan_create_interleaved(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, p1, p2,
                                                   components_, batch_, allocate ? 1 : 0, &plan));
        else if (data_) {
            const size_t m[3] = {data_->Nx, data_->Ny, data_->Nz};
            const size_t k[3] = {spectral_ ? spectral_->Nx : gs->Nx, spectral_ ? spectral_->Ny : gs->Ny, spectral_ ? spectral_->Nz : gs->Nz};
            DFFT_CALL(dfft_plan_create_pruned(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, m, k, p1, p2, batch_,
                                              allocate ? 1 : 0, &plan));
        } else if (spectral_)
            DFFT_CALL(dfft_plan_create_padded(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, spectral_->Nx, spectral_->Ny,
                                              spectral_->Nz, p1, p2, batch_, allocate ? 1 : 0, &plan));
        else if (per_axis)
            DFFT_CALL(dfft_plan_create_r2r(comm, &c, decomp, dfft_shim::prec<T>::value, kinds, gs->Nx, gs->Ny, gs->Nz, p1, p2, batch_,
                                           inplace_ ? 1 : 0, allocate ? 1 : 0, &plan));
        else if (inplace_)
            DFFT_CALL(dfft_plan_create_inplace(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, p1, p2, batch_,
                                               allocate ? 1 : 0, &plan));
        else if (batch_ == 1)
            DFFT_CALL(dfft_plan_create(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, p1, p2, allocate ? 1 : 0, &plan));
        else
            DFFT_CALL(dfft_plan_create_batched(comm, &c, decomp, dfft_shim::prec<T>::value, transform, gs->Nx, gs->Ny, gs->Nz, p1, p2, batch_,
                                               allocate ? 1 : 0, &plan));
        initialized = true;
    }
    size_t batch_ = 1;       // fields of the plan initFFT is creating
    bool inplace_ = false;   // whether initFFT is creating an in-place plan
    GlobalSize* spectral_ = nullptr;  // the spectrum of the padded (or pruned) plan initFFT is creating
    GlobalSize* data_ = nullptr;      // the data block of the pruned plan initFFT is creating
    size_t components_ = 1;  // values per point of the interleaved plan initFFTInterleaved is creating
    const size_t* in_boxes_ = nullptr;   // the boxes of the box plan initFFT is creating
    const size_t* out_boxes_ = nullptr;
    Configurations config;
    dfft_comm_t comm;
    int transform;
    bool per_axis = false;  // constructed with per-axis kinds
    int kinds[3] = {0, 0, 0};
    int pidx = 0, pcnt = 1;
    dfft_plan_t plan = nullptr;
    bool initialized = false;
};

template <typename T>
class MPIcuFFT_Slab : public MPIcuFFT<T> {
public:
    using MPIcuFFT<T>::MPIcuFFT;
    using MPIcuFFT<T>::initFFT;
    void initFFT(GlobalSize* global_size, Partition* /*partition*/, bool allocate = true) override {
        this->create(DFFT_SLAB_ZY_THEN_X, global_size, size_t(this->pcnt), 1, allocate);
    }
    void initFFT(GlobalSize* global_size, bool allocate = true) { initFFT(global_size, nullptr, allocate); }
    void execR2C(void* out, const void* in) override { if (!this->initialized) return; DFFT_CALL(dfft_exec_r2c(this->plan, out, in)); }
    virtual void execC2R(void* out, const void* in) { if (!this->initialized) return; DFFT_CALL(dfft_exec_c2r(this->plan, out, in)); }
    // not in the reference: complex transform (plan constructed with transform_ = DFFT_C2C)
    virtual void execC2C(void* out, const void* in, int direction) { DFFT_CALL(dfft_exec_c2c(this->plan, out, in, direction)); }
};

template <typename T>
class MPIcuFFT_Slab_Z_Then_YX : public MPIcuFFT_Slab<T> {
public:
    using MPIcuFFT_Slab<T>::MPIcuFFT_Slab;
    using MPIcuFFT_Slab<T>::initFFT;
    void initFFT(GlobalSize* global_size, Partition* /*partition*/, bool allocate = true) override {
        this->create(DFFT_SLAB_Z_THEN_YX, global_size, size_t(this->pcnt), 1, allocate);
    }
    // the override above hides the base's two-argument form (mpicufft_slab_z_then_yx.hpp:34-35 declares both)
    void initFFT(GlobalSize* global_size, bool allocate = true) { initFFT(global_size, nullptr, allocate); }
};

template <typename T>
class MPIcuFFT_Pencil : public MPIcuFFT<T> {
public:
    using MPIcuFFT<T>::MPIcuFFT;
    using MPIcuFFT<T>::initFFT;
    void initFFT(GlobalSize* global_size, Partition* partition, bool allocate = true) override {
        if (partition == nullptr || global_size == nullptr) throw std::runtime_error("GlobalSize or Partition not initialized!");
        if (partition->P1 * partition->P2 != size_t(this->pcnt)) throw std::runtime_error("Invalid Input Partition!");
        gs_ = *global_size; part_ = *partition;
        this->create(DFFT_PENCIL, global_size, partition->P1, partition->P2, allocate);
    }
    void execR2C(void* out, const void* in) override { execR2C(out, in, 3); }
    virtual void execC2R(void* out, const void* in) { execC2R(out, in, 3); }
    virtual void execR2C(void* out, const void* in, int d) {
        if (!this->initialized) throw std::runtime_error("cuFFT plans are not yet initialized!");
        DFFT_CALL(dfft_exec_r2c_partial(this->plan, out, in, d));
    }
    virtual void execC2R(void* out, const void* in, int d) {
        if (!this->initialized) throw std::runtime_error("cuFFT plans are not yet initialized!");
        DFFT_CALL(dfft_exec_c2r_partial(this->plan, out, in, d));
    }
    virtual void execC2C(void* out, const void* in, int direction, int d = 3) { DFFT_CALL(dfft_exec_c2c_partial(this->plan, out, in, direction, d)); }
    // getPartitionDimensions(input_dim, transposed_dim, output_dim) — mpicufft_pencil.hpp:112-116
    void getPartitionDimensions(Partition_Dimensions& in_, Partition_Dimensions& tr_, Partition_Dimensions& out_) {
        const size_t nzc = this->transform == DFFT_R2C ? gs_.Nz / 2 + 1 : gs_.Nz;
        auto fill = [](std::vector<size_t>& size, std::vector<size_t>& start, size_t n, size_t parts) {
            size.resize(parts); start.resize(parts);
            dfft_partition(n, parts, size.data(), start.data());
        };
        fill(in_.size_x, in_.start_x, gs_.Nx, part_.P1); fill(in_.size_y, in_.start_y, gs_.Ny, part_.P2); fill(in_.size_z, in_.start_z, gs_.Nz, 1);
        fill(tr_.size_x, tr_.start_x, gs_.Nx, part_.P1); fill(tr_.size_y, tr_.start_y, gs_.Ny, 1); fill(tr_.size_z, tr_.start_z, nzc, part_.P2);
        fill(out_.size_x, out_.start_x, gs_.Nx, 1); fill(out_.size_y, out_.start_y, gs_.Ny, part_.P1); fill(out_.size_z, out_.start_z, nzc, part_.P2);
    }

private:
    GlobalSize gs_{1, 1, 2};
    Partition part_{1, 1};
};

// "Realigned" variants (/root/reference/include/mpicufft_slab_opt1.hpp, mpicufft_slab_z_then_yx_opt1.hpp,
// mpicufft_pencil_opt1.hpp): in the reference they make cuFFT store transposed so that the send side is contiguous;
// results and output layouts are identical to the default classes.  Here the transposing store is always fused into
// the FFT passes, so the names are aliases.
template <typename T> using MPIcuFFT_Slab_Opt1 = MPIcuFFT_Slab<T>;
template <typename T> using MPIcuFFT_Slab_Z_Then_YX_Opt1 = MPIcuFFT_Slab_Z_Then_YX<T>;
template <typename T> using MPIcuFFT_Pencil_Opt1 = MPIcuFFT_Pencil<T>;
