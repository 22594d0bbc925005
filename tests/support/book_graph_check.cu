// Host twin of rz_openings_book_graph: the levels built by the expansion step of csrc/rz_openings.cuh with the dedupe
// done by a stable sort on the canonical key (as tests/support/openings_check.cu does), then book_edges() per node.
//   argv[1] = plies; argv[2], argv[3] (optional) = own, enemy of level 0 in decimal (default the initial position).
//   Prints "counts c_0 .. c_plies", then one line per node, level by level in ascending canonical-key order:
//   "own enemy k sq_1 child_1 .. sq_k child_k" (bitboards in decimal, mover's frame; k = 0 on the last level).
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
    const u64 root_own = argc > 3 ? strtoull(argv[2], nullptr, 10) : kStartBlack;
    const u64 root_enemy = argc > 3 ? strtoull(argv[3], nullptr, 10) : kStartWhite;
    std::vector<std::vector<u64>> own{{root_own}}, enemy{{root_enemy}};
    for (int level = 0; level < plies; ++level) {
        const std::vector<u64>&o = own[level], &e = enemy[level];
        std::vector<Child> ch;
        for (size_t i = 0; i < o.size(); ++i)
            for (u64 m = find_correct_moves(o[i], e[i]); m; m &= m - 1) {
                u64 co, ce;
                if (!child(o[i], e[i], ctz64(m), co, ce)) continue;
                Child c{0, 0, i, ctz64(m)};
                canonical(co, ce, c.hi, c.lo);
                ch.push_back(c);
            }
        std::stable_sort(ch.begin(), ch.end(), [](const Child& a, const Child& b) { return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo); });
        std::vector<u64> own2, enemy2;
        for (size_t j = 0; j < ch.size(); ++j) {
            if (j > 0 && ch[j].hi == ch[j - 1].hi && ch[j].lo == ch[j - 1].lo) continue;
            u64 co, ce;
            child(o[ch[j].parent], e[ch[j].parent], ch[j].sq, co, ce);
            own2.push_back(co);
            enemy2.push_back(ce);
        }
        own.push_back(own2);
        enemy.push_back(enemy2);
    }
    printf("counts");
    for (const auto& lv : own) printf(" %zu", lv.size());
    printf("\n");
    for (int level = 0; level <= plies; ++level) {
        std::vector<u64> hi, lo;
        if (level < plies)
            for (size_t j = 0; j < own[level + 1].size(); ++j) {
                u64 h, l;
                canonical(own[level + 1][j], enemy[level + 1][j], h, l);
                hi.push_back(h);
                lo.push_back(l);
            }
        for (size_t i = 0; i < own[level].size(); ++i) {
            uint8_t sq[64];
            int32_t idx[64];
            const int k = level < plies ? book_edges(own[level][i], enemy[level][i], hi.data(), lo.data(), hi.size(), sq, idx) : 0;
            printf("%llu %llu %d", (unsigned long long)own[level][i], (unsigned long long)enemy[level][i], k);
            for (int j = 0; j < k; ++j) printf(" %d %d", sq[j], idx[j]);
            printf("\n");
        }
    }
    return 0;
}
