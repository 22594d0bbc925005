// Host-side run of the deep solver's leaf machine with its transposition table (csrc/rz_solver_deep.cuh is host/device
// code).  argv[1] = buckets of the table (0: no table), argv[2] = node steps between suspensions (0: each question runs
// to its answer in one call; n > 0: the machine is parked every n steps and resumed, as the kernel does at the end of a
// slice).  Reads commands, one per line (positions in hex, own to move):
//   Q own enemy t           the leaf question "value >= t?" as a lane of deep_slice_kernel asks it: prints 0 or 1
//   S own enemy t r move    store the answer r of "value >= t" (and its proving move, or -1): prints nothing
//   L own enemy             prints "lo hi move" of the position's entry, or "miss"
//   P                       prints "steps N suspensions N lookups N cutoffs N hints N stores N replaced N merges N dropped N"
//   X                       empties the table and zeroes every count
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "rz_solver_deep.cuh"
using namespace rz;
using namespace rz::deep;

int main(int argc, char** argv) {
    const unsigned long long buckets = argc > 1 ? strtoull(argv[1], nullptr, 10) : 0;
    const int every = argc > 2 ? atoi(argv[2]) : 0;
    if (buckets & (buckets - 1)) { fprintf(stderr, "buckets must be a power of two\n"); return 2; }
    std::vector<TableEntry> entries(buckets * kTableWays);
    TableLane tl;
    tl.tab.entries = entries.data();
    tl.tab.mask = buckets ? buckets - 1 : 0;
    NoTable none;
    long long steps = 0, suspensions = 0;
    auto reset = [&] {
        memset(entries.data(), 0, entries.size() * sizeof(TableEntry));
        memset(tl.cnt, 0, sizeof(tl.cnt));
        steps = suspensions = 0;
    };
    reset();
    LeafFrame stk[kLeafStack];
    char cmd[8];
    while (scanf("%7s", cmd) == 1) {
        unsigned long long own = 0, enemy = 0;
        int t = 0, r = 0, move = -1;
        if (cmd[0] == 'Q' && scanf("%llx %llx %d", &own, &enemy, &t) == 3) {
            int depth;
            leaf_init(stk, depth, own, enemy, t);
            int res = buckets ? tl.enter(stk[0]) : -1;
            while (res < 0 || res == kLeafSuspended) {
                res = buckets ? leaf_advance(stk, depth, steps, every ? every : 1 << 30, tl, [] { return false; })
                              : leaf_advance(stk, depth, steps, every ? every : 1 << 30, none, [] { return false; });
                suspensions += res == kLeafSuspended;
            }
            printf("%d\n", res);
        } else if (cmd[0] == 'S' && buckets && scanf("%llx %llx %d %d %d", &own, &enemy, &t, &r, &move) == 5) {
            tl.store(own, enemy, t, r != 0, move);
        } else if (cmd[0] == 'L' && buckets && scanf("%llx %llx", &own, &enemy) == 2) {
            int lo, hi, mv;
            if (table_lookup(tl.tab, own, enemy, lo, hi, mv)) printf("%d %d %d\n", lo, hi, mv);
            else printf("miss\n");
        } else if (cmd[0] == 'P') {
            printf("steps %lld suspensions %lld lookups %u cutoffs %u hints %u stores %u replaced %u merges %u dropped %u\n",
                   steps, suspensions, tl.cnt[kTabLookups], tl.cnt[kTabCutoffs], tl.cnt[kTabHints], tl.cnt[kTabStores],
                   tl.cnt[kTabReplaced], tl.cnt[kTabMerges], tl.cnt[kTabDropped]);
        } else if (cmd[0] == 'X') {
            reset();
        } else {
            fprintf(stderr, "bad command %s\n", cmd);
            return 2;
        }
    }
    return 0;
}
