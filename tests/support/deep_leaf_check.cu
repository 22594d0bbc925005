// Host-side run of the deep solver's leaf machine (csrc/rz_solver_deep.cuh is host/device code): reads lines
// "own enemy t" (hex hex int), prints "0" or "1" = (value >= t).  argv[1] = node steps between suspensions (0: each
// question runs to its answer in one call; n > 0: the machine is parked every n steps and resumed, as the kernel does at
// the end of a slice).  Prints the number of suspensions to stderr.
#include <cstdio>
#include <cstdlib>
#include "rz_solver_deep.cuh"
using namespace rz;
using namespace rz::deep;
int main(int argc, char** argv) {
    const int every = argc > 1 ? atoi(argv[1]) : 0;
    unsigned long long own, enemy;
    int t;
    long long suspensions = 0;
    LeafFrame stk[kLeafStack];
    while (scanf("%llx %llx %d", &own, &enemy, &t) == 3) {
        int depth;
        leaf_init(stk, depth, own, enemy, t);
        long long steps = 0;
        int r;
        while ((r = leaf_advance(stk, depth, steps, every ? every : 1 << 30, [] { return false; })) == kLeafSuspended)
            ++suspensions;
        printf("%d\n", r);
    }
    fprintf(stderr, "suspensions %lld\n", suspensions);
    return 0;
}
