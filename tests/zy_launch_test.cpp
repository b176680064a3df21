// Host check of zy_launch_of (distributedfft_b200/csrc/zy_order.hpp): the fused z + y kernel derives its launch's
// counter base and epoch from a CTA's first draw.  Several launches of one step draw from one counter that is never
// reset, with the CTAs' draws interleaved in a pseudo-random order; every draw's (epoch, ticket) must equal what
// host bookkeeping of the base (advanced by total + grid after each launch) and of the epoch gives.
#include <cstdio>
#include <vector>

#include "../distributedfft_b200/csrc/zy_order.hpp"

using dfft::ZyLaunch;
using dfft::ZyOrder;

static int fails = 0;
#define CHECK(c, ...)                                  \
    do {                                               \
        if (!(c)) {                                    \
            if (fails < 20) std::printf(__VA_ARGS__);  \
            ++fails;                                   \
        }                                              \
    } while (0)

static unsigned long long rng = 88172645463325252ull;
static unsigned next_rand() {
    rng ^= rng << 13;
    rng ^= rng >> 7;
    rng ^= rng << 17;
    return unsigned(rng >> 32);
}

static void check(int nx, int gpp, int na, int nb, int ahead, int grid, int launches) {
    const ZyOrder o{nx, gpp, na, nb, ahead};
    const long long total = o.total();
    const unsigned long long K = o.draws(unsigned(grid));
    CHECK(K == (unsigned long long)(total + grid), "nx=%d gpp=%d grid=%d: draws %llu\n", nx, gpp, grid, K);
    unsigned long long ctr = 0;                       // the device counter
    unsigned long long old_base = 0, old_epoch = 0;   // the host bookkeeping the kernel used to receive
    for (int l = 0; l < launches; ++l) {
        ++old_epoch;
        std::vector<int> active(grid, 1);
        std::vector<unsigned long long> base(grid, 0), epoch(grid, 0);
        std::vector<int> started(grid, 0);
        int running = grid;
        long long drawn = 0;
        while (running) {
            const int c = int(next_rand() % unsigned(grid));
            if (!active[c]) continue;
            const unsigned long long raw = ctr++;
            if (!started[c]) {  // the CTA's first draw fixes its launch
                const ZyLaunch z = dfft::zy_launch_of(raw, K);
                base[c] = z.base;
                epoch[c] = z.epoch;
                started[c] = 1;
            }
            const long long ticket = (long long)(raw - base[c]);
            CHECK(base[c] == old_base && epoch[c] == old_epoch && ticket == (long long)(raw - old_base),
                  "nx=%d gpp=%d L=%d grid=%d launch %d: raw %llu -> epoch %llu ticket %lld, expected epoch %llu ticket %lld\n", nx, gpp,
                  ahead, grid, l, raw, epoch[c], ticket, old_epoch, (long long)(raw - old_base));
            ++drawn;
            if (ticket >= total) {
                active[c] = 0;
                --running;
            }
        }
        CHECK((unsigned long long)drawn == K, "nx=%d gpp=%d grid=%d launch %d: drew %lld, expected %llu\n", nx, gpp, grid, l, drawn, K);
        old_base += (unsigned long long)(total + grid);
    }
    // every raw value of the launches, directly
    for (unsigned long long raw = 0; raw < ctr; ++raw) {
        const ZyLaunch z = dfft::zy_launch_of(raw, K);
        CHECK(z.epoch == raw / K + 1 && z.base <= raw && raw - z.base < K && z.base % K == 0, "K=%llu raw=%llu\n", K, raw);
    }
}

int main() {
    const int cases[][4] = {
        // nx, planes per group, phase-A items per plane, phase-B items per plane
        {512, 1, 64, 64}, {256, 1, 32, 32}, {64, 1, 64, 64}, {1024, 1, 16, 16}, {64, 12, 32, 64}, {7, 2, 5, 3}, {1, 1, 4, 4}, {13, 5, 1, 1},
    };
    for (const auto& c : cases)
        for (int ahead : {1, 3})
            for (int grid : {1, 3, 264}) check(c[0], c[1], c[2], c[3], ahead, grid, 4);
    std::printf("fails=%d\n", fails);
    return fails != 0;
}
