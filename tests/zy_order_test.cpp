// Host check of the fused z + y stage's work list (distributedfft_b200/csrc/zy_order.hpp, the header the kernel
// decodes its tickets with): every item issued exactly once, in its group, every dependency on a lower ticket, the
// look-ahead, and the per-group counter targets of consecutive launches (epochs) reached exactly by that launch's items.
#include <cstdio>
#include <vector>

#include "../distributedfft_b200/csrc/zy_order.hpp"

using dfft::ZyItem;
using dfft::ZyOrder;

static int fails = 0;
#define CHECK(c, ...)                                  \
    do {                                               \
        if (!(c)) {                                    \
            if (fails < 20) std::printf(__VA_ARGS__);  \
            ++fails;                                   \
        }                                              \
    } while (0)

static void check(int nx, int gpp, int na, int nb, int ahead, int grid) {
    const ZyOrder o{nx, gpp, na, nb, ahead};
    const long long total = o.total();
    const int n = o.groups();
    std::vector<int> seen_a(size_t(nx) * na, 0), seen_b(size_t(nx) * nb, 0);
    std::vector<long long> last_a(n, -1), first_b(n, total);
    for (long long t = 0; t < total; ++t) {
        const ZyItem it = o.decode(t);
        CHECK(it.group >= 0 && it.group < n, "nx=%d gpp=%d: ticket %lld -> group %d\n", nx, gpp, t, it.group);
        if (it.group < 0 || it.group >= n) continue;
        const int per = it.phase == 0 ? na : nb;
        CHECK(it.tile >= 0 && it.tile < (long long)nx * per, "nx=%d gpp=%d: ticket %lld -> tile %lld\n", nx, gpp, t, it.tile);
        if (it.tile < 0 || it.tile >= (long long)nx * per) continue;
        CHECK(int(it.tile / per) / gpp == it.group, "nx=%d gpp=%d: ticket %lld: tile %lld is not in group %d\n", nx, gpp, t, it.tile, it.group);
        if (it.phase == 0) {
            seen_a[it.tile]++;
            last_a[it.group] = t;
        } else {
            seen_b[it.tile]++;
            if (t < first_b[it.group]) first_b[it.group] = t;
        }
    }
    for (size_t i = 0; i < seen_a.size(); ++i) CHECK(seen_a[i] == 1, "nx=%d gpp=%d: phase-A tile %zu issued %d times\n", nx, gpp, i, seen_a[i]);
    for (size_t i = 0; i < seen_b.size(); ++i) CHECK(seen_b[i] == 1, "nx=%d gpp=%d: phase-B tile %zu issued %d times\n", nx, gpp, i, seen_b[i]);
    long long a_sum = 0;
    for (int g = 0; g < n; ++g) {
        // dependencies point to lower tickets: the last A item of g precedes the first B item of g
        CHECK(last_a[g] < first_b[g], "nx=%d gpp=%d: group %d: B starts at ticket %lld before A ends at %lld\n", nx, gpp, g, first_b[g], last_a[g]);
        // look-ahead of exactly L groups: A(g+L) is issued before B(g), A(g+L+1) after it
        if (g + ahead < n) CHECK(last_a[g + ahead] < first_b[g], "nx=%d gpp=%d L=%d: A(%d) not ahead of B(%d)\n", nx, gpp, ahead, g + ahead, g);
        if (g + ahead + 1 < n) CHECK(first_b[g] < last_a[g + ahead + 1], "nx=%d gpp=%d L=%d: B(%d) behind A(%d)\n", nx, gpp, ahead, g, g + ahead + 1);
        a_sum += o.a_items(g);
    }
    CHECK(a_sum == (long long)nx * na, "nx=%d gpp=%d: a_items sum %lld\n", nx, gpp, a_sum);
    // Three launches of `grid` CTAs: the ticket counter and the group counters are never reset.  A CTA draws until it
    // gets a ticket >= total (one extra draw per CTA), so a launch advances the ticket counter by total + grid; the
    // group counter of g reaches epoch * a_items(g) exactly when the last A item of g in that launch has finished.
    unsigned long long ctr = 0, base = 0;
    std::vector<unsigned long long> done(n, 0);
    for (unsigned long long epoch = 1; epoch <= 3; ++epoch) {
        std::vector<int> active(grid, 1);
        int running = grid;
        while (running) {
            for (int c = 0; c < grid; ++c) {
                if (!active[c]) continue;
                const long long t = (long long)(ctr++ - base);
                if (t >= total) { active[c] = 0; --running; continue; }
                const ZyItem it = o.decode(t);
                if (it.phase == 1) {
                    CHECK(done[it.group] >= epoch * (unsigned long long)o.a_items(it.group),
                          "nx=%d gpp=%d epoch %llu: B item of group %d runs before its A items finished\n", nx, gpp, epoch, it.group);
                } else {
                    ++done[it.group];
                    CHECK(done[it.group] <= epoch * (unsigned long long)o.a_items(it.group), "nx=%d gpp=%d: group %d counter overshoots\n", nx, gpp, it.group);
                }
            }
        }
        CHECK(ctr - base == (unsigned long long)(total + grid), "nx=%d gpp=%d: launch drew %llu tickets, expected %lld\n", nx, gpp, ctr - base, total + grid);
        for (int g = 0; g < n; ++g)
            CHECK(done[g] == epoch * (unsigned long long)o.a_items(g), "nx=%d gpp=%d epoch %llu: group %d counter %llu\n", nx, gpp, epoch, g, done[g]);
        base = ctr;
    }
}

int main() {
    const int cases[][4] = {
        // nx, planes per group, phase-A items per plane, phase-B items per plane
        {512, 1, 64, 64}, {512, 2, 64, 64}, {512, 3, 64, 64}, {64, 12, 32, 64}, {1024, 8, 16, 16},
        {7, 2, 5, 3},     {7, 7, 5, 3},     {7, 8, 5, 3},     {1, 1, 4, 4},     {2, 1, 3, 5},     {5, 4, 2, 9}, {13, 5, 1, 1},
    };
    for (const auto& c : cases)
        for (int ahead : {1, 2, 3, 9})
            for (int grid : {1, 3, 264}) check(c[0], c[1], c[2], c[3], ahead, grid);
    std::printf("fails=%d\n", fails);
    return fails != 0;
}
