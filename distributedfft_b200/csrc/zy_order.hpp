// zy_order.hpp — work list of the fused two-phase kernel (fft_zy_fused_kernel in fft_kernels.cuh).
//
// The array is nx planes; the planes are cut into groups of `gpp` consecutive planes (the last group may be shorter).
// Phase A has `na` work items (CTA tiles) per plane, phase B `nb`; the B items of a group read what the A items of the
// same group wrote.  CTAs draw tickets 0, 1, 2, ... from one global counter, and ticket order is, with a look-ahead of
// L groups (n = number of groups):
//
//     A(0), ..., A(L-1),  A(L), B(0),  A(L+1), B(1),  ...,  A(n-1), B(n-1-L),  B(n-L), ..., B(n-1)
//
// Phase A runs L groups ahead of phase B: while the B items of group g run, the A items of group g+L fill the L2 with
// what B(g+L) will read.  The look-ahead is what keeps a B item from waiting: the items of A(g) are drawn L groups of
// work before the first item of B(g), so with L * gpp * (na + nb) above the number of resident CTAs they have finished
// by then.  Every B item of group g depends on all A items of group g, whose tickets are all lower than any ticket of
// B(g) — the property the deadlock argument at the wait in ticket_loop (fft_kernels.cuh) rests on.
//
// Host-compiled as well (tests/zy_order_test.cpp checks the list).
#pragma once

#if defined(__CUDACC__)
#define DFFT_ZY_HD __host__ __device__ __forceinline__
#else
#define DFFT_ZY_HD inline
#endif

namespace dfft {

struct ZyItem {
    int phase;       // 0 = phase A, 1 = phase B
    int group;       // plane group
    long long tile;  // tile index within the phase, over the whole array (plane x owns tiles [x*na, (x+1)*na) of phase A)
};

struct ZyOrder {
    int nx, gpp, na, nb;
    int ahead;  // look-ahead L in groups (>= 1)

    DFFT_ZY_HD int groups() const { return (nx + gpp - 1) / gpp; }
    DFFT_ZY_HD int planes(int g) const { return nx - g * gpp < gpp ? nx - g * gpp : gpp; }
    // phase-A items of group g: the number of completions a B item of g waits for (per exec)
    DFFT_ZY_HD long long a_items(int g) const { return (long long)planes(g) * na; }
    DFFT_ZY_HD long long total() const { return (long long)nx * (na + nb); }

    // ticket (0 <= t < total()) -> work item
    DFFT_ZY_HD ZyItem decode(long long t) const {
        const int n = groups();
        const int L = ahead < n ? ahead : n;
        const long long fa = (long long)gpp * na, fb = (long long)gpp * nb;  // items of a full group
        // A(0..L-1): A tiles 0 .. in order (a short last group only when L == n)
        const long long a_pre = L == n ? (long long)nx * na : L * fa;
        if (t < a_pre) return ZyItem{0, int(t / fa), t};
        t -= a_pre;
        // pairs (A(i), B(i-L)) of two full groups: i = L .. n-2
        const long long full_pairs = n - 1 - L > 0 ? n - 1 - L : 0;
        const long long q = t / (fa + fb);
        if (q < full_pairs) {
            const int i = L + int(q);
            const long long r = t - q * (fa + fb);
            if (r < fa) return ZyItem{0, i, i * fa + r};
            return ZyItem{1, i - L, (i - L) * fb + (r - fa)};
        }
        t -= full_pairs * (fa + fb);
        if (n > L) {  // the last pair: A(n-1) may be a short group
            const int i = n - 1;
            const long long ai = a_items(i);
            if (t < ai) return ZyItem{0, i, i * fa + t};
            t -= ai;
            if (t < fb) return ZyItem{1, i - L, (i - L) * fb + t};
            t -= fb;
        }
        // B(n-L .. n-1), in order
        const long long tile = (n - L) * fb + t;
        return ZyItem{1, int(tile / fb), tile};
    }

    // Tickets one launch of `grid` CTAs draws from the counter: every ticket below total() once, and one more per CTA,
    // which tells it to stop.
    DFFT_ZY_HD unsigned long long draws(unsigned grid) const { return (unsigned long long)total() + grid; }
};

// Which launch a raw counter value belongs to.  The counter is zeroed once and never reset, and every launch of a step
// has the same grid, so launch e (from 1) draws exactly the values [(e - 1) * K, e * K) with K = draws(grid), once the
// launches before it have ended (launches of one step are stream-ordered).  A CTA's first draw therefore fixes the
// launch's base and epoch without any value from the host, which is what lets a captured graph replay the launch.
struct ZyLaunch {
    unsigned long long base;   // counter value of the launch's ticket 0
    unsigned long long epoch;  // launches of this step so far, this one included
};
DFFT_ZY_HD ZyLaunch zy_launch_of(unsigned long long raw, unsigned long long draws_per_launch) {
    const unsigned long long e = raw / draws_per_launch;
    return ZyLaunch{e * draws_per_launch, e + 1};
}

}  // namespace dfft
