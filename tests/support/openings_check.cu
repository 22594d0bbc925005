// Host twin of rz_openings_enumerate: the expansion step of csrc/rz_openings.cuh compiled for the host, with the dedupe
// done by a stable sort on the canonical key.
//   argv[1] = plies.  Prints "counts c_0 .. c_plies", then one line per opening in ascending canonical-key order:
//   "own enemy m_1 .. m_plies" (bitboards in decimal, mover's frame).
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "rz_openings.cuh"
using namespace rz;
using namespace rz::openings;

struct Child { u64 hi, lo; size_t parent; int sq; };

int main(int argc, char** argv) {
    const int plies = argc > 1 ? atoi(argv[1]) : 1;
    std::vector<u64> own{kStartBlack}, enemy{kStartWhite};
    std::vector<std::vector<int>> moves{{}};
    std::vector<size_t> counts{1};
    for (int level = 0; level < plies; ++level) {
        std::vector<Child> ch;
        for (size_t i = 0; i < own.size(); ++i)
            for (u64 m = find_correct_moves(own[i], enemy[i]); m; m &= m - 1) {
                u64 co, ce;
                if (!child(own[i], enemy[i], ctz64(m), co, ce)) continue;
                Child c{0, 0, i, ctz64(m)};
                canonical(co, ce, c.hi, c.lo);
                ch.push_back(c);
            }
        std::stable_sort(ch.begin(), ch.end(), [](const Child& a, const Child& b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); });
        std::vector<u64> own2, enemy2;
        std::vector<std::vector<int>> moves2;
        for (size_t j = 0; j < ch.size(); ++j) {
            if (j > 0 && ch[j].hi == ch[j - 1].hi && ch[j].lo == ch[j - 1].lo) continue;
            u64 co, ce;
            child(own[ch[j].parent], enemy[ch[j].parent], ch[j].sq, co, ce);
            own2.push_back(co);
            enemy2.push_back(ce);
            moves2.push_back(moves[ch[j].parent]);
            moves2.back().push_back(ch[j].sq);
        }
        own.swap(own2); enemy.swap(enemy2); moves.swap(moves2);
        counts.push_back(own.size());
    }
    printf("counts");
    for (size_t c : counts) printf(" %zu", c);
    printf("\n");
    for (size_t i = 0; i < own.size(); ++i) {
        printf("%llu %llu", (unsigned long long)own[i], (unsigned long long)enemy[i]);
        for (int sq : moves[i]) printf(" %d", sq);
        printf("\n");
    }
    return 0;
}
