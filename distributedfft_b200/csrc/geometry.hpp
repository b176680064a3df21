// geometry.hpp — host-only partition / layout arithmetic of a plan (no CUDA).
//
// Restates the split rule of the reference's initFFT:
//   slab   /root/reference/src/slab/default/mpicufft_slab.cpp:112-128   (x split -> y split)
//   z_yx   /root/reference/src/slab/z_then_yx/mpicufft_slab_z_then_yx.cpp (x split -> z split)
//   pencil /root/reference/src/pencil/mpicufft_pencil.cpp:84-110         (pidx = i*P2 + j)
// size[p] = n/parts + (p < n%parts); start = prefix sum.
#pragma once
#include <algorithm>
#include <cstddef>
#include <vector>

#include "../../include/dfft.h"

namespace dfft {

struct Split {
    std::vector<size_t> size, start;
    void make(size_t n, size_t parts) {
        size.assign(parts, n / parts);
        for (size_t p = 0; p < n % parts; ++p) size[p]++;
        start.assign(parts, 0);
        for (size_t p = 1; p < parts; ++p) start[p] = start[p - 1] + size[p - 1];
    }
};

// A box of grid points [lo, hi) per axis (x, y, z), the unit of dfft_plan_create_boxes: each rank's caller array is its box,
// dense, z contiguous.
struct Box {
    size_t lo[3] = {0, 0, 0}, hi[3] = {0, 0, 0};
    static Box of(const size_t size[3], const size_t start[3]) {
        Box b;
        for (int a = 0; a < 3; ++a) { b.lo[a] = start[a]; b.hi[a] = start[a] + size[a]; }
        return b;
    }
    size_t extent(int a) const { return hi[a] > lo[a] ? hi[a] - lo[a] : 0; }
    size_t volume() const { return extent(0) * extent(1) * extent(2); }
    bool operator==(const Box& o) const {
        for (int a = 0; a < 3; ++a)
            if (lo[a] != o.lo[a] || hi[a] != o.hi[a]) return false;
        return true;
    }
    // the common part (volume 0 if there is none)
    Box operator&(const Box& o) const {
        Box b;
        for (int a = 0; a < 3; ++a) { b.lo[a] = std::max(lo[a], o.lo[a]); b.hi[a] = std::max(b.lo[a], std::min(hi[a], o.hi[a])); }
        return b;
    }
    // element offset of grid point p (inside the box) in the box's dense array
    size_t offset(const size_t p[3]) const { return ((p[0] - lo[0]) * extent(1) + (p[1] - lo[1])) * extent(2) + (p[2] - lo[2]); }
};

// Whether `boxes` tile the grid n[0] x n[1] x n[2]: none empty or reaching outside it, no two overlapping, and their
// volumes adding up to the grid's (so that together they cover it).
inline bool tiles(const std::vector<Box>& boxes, const size_t n[3]) {
    size_t total = 0;
    for (size_t i = 0; i < boxes.size(); ++i) {
        const Box& b = boxes[i];
        for (int a = 0; a < 3; ++a)
            if (b.lo[a] >= b.hi[a] || b.hi[a] > n[a]) return false;
        for (size_t j = 0; j < i; ++j)
            if ((b & boxes[j]).volume()) return false;
        total += b.volume();
    }
    return total == n[0] * n[1] * n[2];
}

struct Geometry {
    int decomp = 0, transform = 0;
    size_t nx = 0, ny = 0, nz = 0, nzc = 0;  // nzc: z extent of every complex array (real-to-real: of every real array, Nz)
    // spectral extents (dfft_plan_create_padded): Kx, Ky and the z extent of the spectrum (R2C: Kz/2 + 1); nx, ny, nzc for
    // every other plan.  An axis is padded by the pass that transforms it: the layout after d stages has K on the first d
    // axes in z, y, x order.
    size_t kx = 0, ky = 0, kz = 0, kzc = 0;
    // physical extents of the data (dfft_plan_create_pruned): the field holds Mx x My x Mz points at [0, M) of each axis,
    // zero beyond; nx, ny, nz for every other plan.  The mirror of K: the layout after d stages has M on the axes not yet
    // transformed, and the physical x (pencil: y) split is made over M.
    size_t mx = 0, my = 0, mz = 0;
    int P = 1, P1 = 1, P2 = 1;
    // x split of the input (over P1, or over P for both slab sequences)
    Split sx;
    // pencil: y split of the input over P2;  z split of the spectrum over P2 (z_yx: over P)
    Split sy, sz;
    // y split of the output over P1 (slab zy_x: over P)
    Split oy;

    // returns false on an invalid partition.  kx_, ky_, kz_: the spectral grid, mx_, my_, mz_: the data (0: the physical
    // grid)
    bool init(int decomp_, int transform_, size_t nx_, size_t ny_, size_t nz_, size_t p1, size_t p2, int nranks, size_t kx_ = 0, size_t ky_ = 0,
              size_t kz_ = 0, size_t mx_ = 0, size_t my_ = 0, size_t mz_ = 0) {
        decomp = decomp_; transform = transform_;
        nx = nx_; ny = ny_; nz = nz_;
        const bool real_z = !(transform == DFFT_C2C || transform == DFFT_DCT || transform == DFFT_DST || transform == DFFT_R2HC);
        nzc = real_z ? nz / 2 + 1 : nz;
        kx = kx_ ? kx_ : nx;
        ky = ky_ ? ky_ : ny;
        kz = kz_ ? kz_ : nz;
        kzc = real_z ? kz / 2 + 1 : kz;
        mx = mx_ ? mx_ : nx;
        my = my_ ? my_ : ny;
        mz = mz_ ? mz_ : nz;
        P = nranks;
        if (decomp == DFFT_SLAB_ZY_THEN_X) { P1 = P; P2 = 1; }
        else if (decomp == DFFT_SLAB_Z_THEN_YX) { P1 = P; P2 = 1; }  // P1 only used for the x split
        else if (decomp == DFFT_PENCIL) { P1 = int(p1); P2 = int(p2); }
        else return false;
        if (P1 < 1 || P2 < 1 || size_t(P1) * size_t(P2) != size_t(P)) return false;
        if (nx == 0 || ny == 0 || nz == 0) return false;
        sx.make(mx, P1);
        if (decomp == DFFT_SLAB_Z_THEN_YX) {
            sy.make(my, 1);
            sz.make(kzc, P);
            oy.make(ky, 1);
        } else {
            sy.make(my, P2);
            sz.make(kzc, P2);
            oy.make(ky, P1);
        }
        return true;
    }
    bool padded() const { return kx != nx || ky != ny || kz != nz; }
    bool pruned() const { return mx != nx || my != ny || mz != nz; }
    int pi(int rank) const { return decomp == DFFT_PENCIL ? rank / P2 : rank; }
    int pj(int rank) const { return decomp == DFFT_PENCIL ? rank % P2 : 0; }

    // which: 0 input, 1 after z, 2 after z and y, 3 output
    void layout(int rank, int which, size_t size[3], size_t start[3]) const {
        const int i = pi(rank), j = pj(rank);
        if (decomp == DFFT_SLAB_Z_THEN_YX) {
            if (which <= 1) {
                size[0] = sx.size[i]; size[1] = my; size[2] = which == 0 ? mz : kzc;
                start[0] = sx.start[i]; start[1] = 0; start[2] = 0;
            } else {
                size[0] = which == 2 ? mx : kx; size[1] = ky; size[2] = sz.size[rank];
                start[0] = 0; start[1] = 0; start[2] = sz.start[rank];
            }
            return;
        }
        switch (which) {
            case 0:
            case 1:
                size[0] = sx.size[i]; size[1] = sy.size[j]; size[2] = which == 0 ? mz : kzc;
                start[0] = sx.start[i]; start[1] = sy.start[j]; start[2] = 0;
                break;
            case 2:
                size[0] = sx.size[i]; size[1] = ky; size[2] = sz.size[j];
                start[0] = sx.start[i]; start[1] = 0; start[2] = sz.start[j];
                break;
            default:
                size[0] = kx; size[1] = oy.size[i]; size[2] = sz.size[j];
                start[0] = 0; start[1] = oy.start[i]; start[2] = sz.start[j];
                break;
        }
    }
    // complex elements of the largest per-rank stage array (the reference's domainsize / sizeof(C_t),
    // mpicufft_slab.cpp:132).  Padded and pruned plans have more: the y pass' physical side [x_i][My][z_j] and the x pass'
    // physical side [Mx][y_i][z_j] (y spectral).  Z_Then_YX holds its y and x passes in one slot of [X][Y][z_r] planes, X
    // and Y the larger of M and K (the forward y pass runs in place, from My to Ky rows; the inverse one from Kx planes),
    // and its first transposition moves zyx_rows rows per x plane.
    // In every other plan they are layouts 2 and 3.
    size_t domain_elems(int rank) const {
        size_t m = 0;
        for (int w = 1; w <= 3; ++w) {
            size_t s[3], o[3];
            layout(rank, w, s, o);
            m = std::max(m, s[0] * s[1] * s[2]);
        }
        if (decomp == DFFT_SLAB_Z_THEN_YX)  // and the all-to-all staging of the z pass's output, [x_i][zyx_rows][Kzc]
            return std::max(m, std::max(std::max(mx, kx) * zyx_rows() * sz.size[rank], sx.size[pi(rank)] * zyx_rows() * kzc));
        const size_t zr = sz.size[pj(rank)];
        return std::max(m, std::max(sx.size[pi(rank)] * my * zr, mx * oy.size[pi(rank)] * zr));
    }
    // Z_Then_YX: rows of the y-pass planes in its slot, both sides of the in-place forward y pass (My in, Ky out)
    size_t zyx_rows() const { return std::max(my, ky); }
};

}  // namespace dfft
