// Host-side checks of the deep solver's forest logic (csrc/rz_solver_deep.cuh is host/device code).
//   argv[1] = "roots": every status pattern (open / TRUE / FALSE) of 1..4 roots under every question: each root's wanted
//     answer 0 or 1 (the move forest of rz_solve_deep), and kEveryRoot on every root (rz_solve_deep_moves).  Prints one
//     line per case: "n status... flip... answered".
//   argv[1] = "moves": reads lines "n_best k v_1 .. v_k" (the true values of k moves) and runs the rounds of
//     rz_solve_deep_moves with plan_round, each root answered from the true value as the forest would.  Prints
//     "rounds lo_1 hi_1 .. lo_k hi_k" per line.
#include <cstdio>
#include <cstring>
#include "rz_solver_deep.cuh"
using namespace rz;
using namespace rz::deep;

int main(int argc, char** argv) {
    if (argc > 1 && !strcmp(argv[1], "roots")) {
        for (int n = 1; n <= 4; ++n) {
            int n_status = 1;
            for (int i = 0; i < n; ++i) n_status *= 3;
            for (int sp = 0; sp < n_status; ++sp)
                for (int fp = 0; fp <= (1 << n); ++fp) {  // fp == 1 << n: kEveryRoot on every root
                    int32_t status[4];
                    Node nodes[4];
                    for (int i = 0, x = sp; i < n; ++i, x /= 3) {
                        status[i] = x % 3;
                        nodes[i] = Node{};
                        nodes[i].parent = -1;
                        nodes[i].flip = (int8_t)(fp == (1 << n) ? kEveryRoot : (fp >> i) & 1);
                    }
                    printf("%d", n);
                    for (int i = 0; i < n; ++i) printf(" %d", status[i]);
                    for (int i = 0; i < n; ++i) printf(" %d", nodes[i].flip);
                    printf(" %d\n", (int)roots_answered(status, nodes, n));
                }
        }
        return 0;
    }
    int n_best, k;
    while (scanf("%d %d", &n_best, &k) == 2) {
        int v[64], lo[64], hi[64], t[64];
        for (int i = 0; i < k; ++i) { if (scanf("%d", &v[i]) != 1) return 2; lo[i] = -64; hi[i] = 64; }
        int rounds = 0;
        for (; rounds < kMaxMoveRounds; ++rounds) {
            if (!plan_round(lo, hi, k, n_best, t)) break;
            for (int i = 0; i < k; ++i) {
                if (t[i] == kNoProbe) continue;
                if (v[i] >= t[i]) lo[i] = t[i] > lo[i] ? t[i] : lo[i]; else hi[i] = t[i] - 1 < hi[i] ? t[i] - 1 : hi[i];
            }
        }
        if (rounds == kMaxMoveRounds && plan_round(lo, hi, k, n_best, t)) rounds = -1;  // more rounds would be needed
        printf("%d", rounds);
        for (int i = 0; i < k; ++i) printf(" %d %d", lo[i], hi[i]);
        printf("\n");
    }
    return 0;
}
