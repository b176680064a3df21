// Host check of the batched stage's work list (ZyOrder with one group per field, as launch_batch_small builds it, from
// distributedfft_b200/csrc/zy_order.hpp): every plane item and slice item of every field issued exactly once, in its
// field, every dependency on a lower ticket, the look-ahead in fields, and — over three launches drawn from one counter
// by interleaved CTAs, each CTA decoding its launch with zy_launch_of from its first draw only — the per-field counter
// targets reached exactly by that launch's phase-A items before any of its phase-B items of the field runs.
#include <cstdio>
#include <vector>

#include "../distributedfft_b200/csrc/zy_order.hpp"

using dfft::ZyItem;
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

static void check(int fields, int items, int ahead, int grid) {
    const ZyOrder o{fields, 1, items, items, ahead};
    const long long total = o.total();
    CHECK(o.groups() == fields && total == 2ll * fields * items, "B=%d: %d groups, %lld items\n", fields, o.groups(), total);
    std::vector<int> seen(size_t(2) * fields * items, 0);
    std::vector<long long> last_a(fields, -1), first_b(fields, total);
    for (long long t = 0; t < total; ++t) {
        const ZyItem it = o.decode(t);
        const bool ok = it.group >= 0 && it.group < fields && it.tile >= 0 && it.tile < (long long)fields * items;
        CHECK(ok, "B=%d: ticket %lld -> field %d item %lld\n", fields, t, it.group, it.tile);
        if (!ok) continue;
        CHECK(it.tile / items == it.group, "B=%d: ticket %lld: item %lld is not in field %d\n", fields, t, it.tile, it.group);
        seen[size_t(it.phase) * fields * items + it.tile]++;
        if (it.phase == 0) last_a[it.group] = t;
        else if (t < first_b[it.group]) first_b[it.group] = t;
    }
    for (size_t i = 0; i < seen.size(); ++i) CHECK(seen[i] == 1, "B=%d: item %zu issued %d times\n", fields, i, seen[i]);
    for (int g = 0; g < fields; ++g) {
        CHECK(last_a[g] < first_b[g], "B=%d: field %d: phase B starts before phase A ends\n", fields, g);
        if (g + ahead < fields) CHECK(last_a[g + ahead] < first_b[g], "B=%d L=%d: field %d not ahead of %d\n", fields, ahead, g + ahead, g);
    }
    // three launches: CTAs draw round-robin from one counter that is never reset; a CTA knows only its first raw draw
    const unsigned long long K = o.draws(unsigned(grid));
    unsigned long long ctr = 0;
    std::vector<unsigned long long> done(fields, 0);
    for (unsigned long long launch = 1; launch <= 3; ++launch) {
        std::vector<int> active(grid, 1);
        std::vector<ZyLaunch> mine(grid);
        std::vector<int> first(grid, 1);
        int running = grid;
        while (running) {
            for (int c = 0; c < grid; ++c) {
                if (!active[c]) continue;
                const unsigned long long raw = ctr++;
                if (first[c]) { mine[c] = dfft::zy_launch_of(raw, K); first[c] = 0; }
                CHECK(mine[c].epoch == launch, "B=%d: CTA %d of launch %llu decodes epoch %llu\n", fields, c, launch, mine[c].epoch);
                const long long t = (long long)(raw - mine[c].base);
                if (t >= total) { active[c] = 0; --running; continue; }
                const ZyItem it = o.decode(t);
                if (it.phase == 1)
                    CHECK(done[it.group] >= launch * (unsigned long long)o.a_items(it.group), "B=%d launch %llu: field %d phase B before phase A\n",
                          fields, launch, it.group);
                else
                    ++done[it.group];
            }
        }
        CHECK(ctr == launch * K, "B=%d: launch %llu drew %llu tickets\n", fields, launch, ctr);
        for (int g = 0; g < fields; ++g)
            CHECK(done[g] == launch * (unsigned long long)o.a_items(g), "B=%d launch %llu: field %d counter %llu\n", fields, launch, g, done[g]);
    }
}

int main() {
    // items per field: 64 at 64^3 (4096-point items), 8 at 32^3
    for (int fields : {1, 2, 3, 8, 64, 257})
        for (int items : {8, 64})
            for (int ahead : {1, 3, 32})
                for (int grid : {1, 5, 264}) check(fields, items, ahead, grid);
    std::printf("fails=%d\n", fails);
    return fails != 0;
}
