// Host twin of rz_openings_book_children: book_children() of csrc/rz_openings.cuh for every node.
//   stdin: "n n_next", then n lines "own enemy" (mover's frame), then n_next lines "key_hi key_lo" (ascending), in decimal.
//   Prints one line per node: "k sq_1 child_1 kind_1 own_1 enemy_1 hi_1 lo_1 .. sq_k child_k kind_k own_k enemy_k hi_k lo_k".
#include <cstdio>
#include <vector>
#include "rz_openings.cuh"
using namespace rz;
using namespace rz::openings;

int main() {
    size_t n = 0, n_next = 0;
    if (scanf("%zu %zu", &n, &n_next) != 2) return 1;
    std::vector<unsigned long long> own(n), enemy(n), hi(n_next), lo(n_next);
    for (size_t i = 0; i < n; ++i)
        if (scanf("%llu %llu", &own[i], &enemy[i]) != 2) return 1;
    for (size_t j = 0; j < n_next; ++j)
        if (scanf("%llu %llu", &hi[j], &lo[j]) != 2) return 1;
    std::vector<u64> next_hi(hi.begin(), hi.end()), next_lo(lo.begin(), lo.end());
    for (size_t i = 0; i < n; ++i) {
        uint8_t sq[64], kind[64];
        int32_t idx[64];
        u64 co[64], ce[64], ch[64], cl[64];
        const int k = book_children(own[i], enemy[i], next_hi.data(), next_lo.data(), n_next, sq, idx, co, ce, ch, cl, kind);
        printf("%d", k);
        for (int j = 0; j < k; ++j)
            printf(" %d %d %d %llu %llu %llu %llu", sq[j], idx[j], kind[j], (unsigned long long)co[j], (unsigned long long)ce[j],
                   (unsigned long long)ch[j], (unsigned long long)cl[j]);
        printf("\n");
    }
    return 0;
}
