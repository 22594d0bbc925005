// rz_openings.cuh -- one expansion step of the opening enumerator, the book graph's edge step and the book's children step
// (rz_openings.cu), __host__ __device__ so that the host checks (tests/support/openings_check.cu, book_graph_check.cu,
// book_children_check.cu) run the same code.
//
// A position is held in the mover's frame (own = the side to move).  Its children are the positions after each legal
// move, again in the new mover's frame; a child whose side to move has no legal move (a pass, or the end of the game) is
// dropped, so every opening the enumerator returns is a sequence of plies without a pass.  Children are numbered in
// (parent index, move square) order, which is the order an exclusive scan of the per-parent counts gives.
#pragma once
#include "rz_bitboard.cuh"

namespace rz {
namespace openings {

// the child of (own, enemy) after the move at sq, in the new mover's frame; false when that mover has no legal move
RZ_HD bool child(u64 own, u64 enemy, int sq, u64& c_own, u64& c_enemy) {
    const u64 fl = calc_flip(sq, own, enemy);
    c_own = enemy ^ fl;
    c_enemy = own | fl | (1ULL << sq);
    return find_correct_moves(c_own, c_enemy) != 0;
}

// the legal moves of (own, enemy) whose child is kept
RZ_HD u64 kept_moves(u64 own, u64 enemy) {
    u64 kept = 0;
    for (u64 m = find_correct_moves(own, enemy); m; m &= m - 1) {
        u64 co, ce;
        if (child(own, enemy, ctz64(m), co, ce)) kept |= m & (~m + 1);
    }
    return kept;
}

// canonical key of a position: the least (own, enemy) pair, compared own first, over its 8 dihedral images
RZ_HD void canonical(u64 own, u64 enemy, u64& k_hi, u64& k_lo) {
    k_hi = own; k_lo = enemy;
    for (int t = 1; t < 8; ++t) {
        const u64 o = dihedral(own, t), e = dihedral(enemy, t);
        if (o < k_hi || (o == k_hi && e < k_lo)) { k_hi = o; k_lo = e; }
    }
}

// the index of key (hi, lo) among the n ascending keys (keys_hi, keys_lo), found by binary search; -1 when it is not there
RZ_HD int32_t find_key(const u64* keys_hi, const u64* keys_lo, size_t n, u64 hi, u64 lo) {
    size_t a = 0, b = n;   // the first key >= (hi, lo)
    while (a < b) {
        const size_t c = (a + b) / 2;
        if (keys_hi[c] < hi || (keys_hi[c] == hi && keys_lo[c] < lo)) a = c + 1;
        else b = c;
    }
    return a < n && keys_hi[a] == hi && keys_lo[a] == lo ? (int32_t)a : -1;
}

// the book graph's edges of (own, enemy) (rz_openings_book_graph): its legal moves in ascending square order, each with
// the index of its child's class among the n_next ascending keys (next_hi, next_lo) of the next level, found by binary
// search; -1 when the child is not an opening (its mover must pass, or the game is over).  -> the number of edges.
RZ_HD int book_edges(u64 own, u64 enemy, const u64* next_hi, const u64* next_lo, size_t n_next, uint8_t* square,
                     int32_t* child_index) {
    int k = 0;
    for (u64 m = find_correct_moves(own, enemy); m; m &= m - 1, ++k) {
        const int sq = ctz64(m);
        square[k] = (uint8_t)sq;
        child_index[k] = -1;
        u64 co, ce, hi, lo;
        if (!child(own, enemy, sq, co, ce)) continue;
        canonical(co, ce, hi, lo);
        child_index[k] = find_key(next_hi, next_lo, n_next, hi, lo);
    }
    return k;
}

// the kind of a child (rz_openings_book_children): an opening, a position whose mover must pass, or a finished game
enum ChildKind : uint8_t { kChildKept = 0, kChildPass = 1, kChildOver = 2 };

// the children of any node (rz_openings_book_children): its legal moves in ascending square order, each with the child
// in the new mover's frame, its canonical key, its kind and the index of its key among the n_next ascending keys (next_hi,
// next_lo) of a sorted level; -1 when the child is not kept or not in that level.  -> the number of children.
RZ_HD int book_children(u64 own, u64 enemy, const u64* next_hi, const u64* next_lo, size_t n_next, uint8_t* square,
                        int32_t* child_index, u64* c_own, u64* c_enemy, u64* c_hi, u64* c_lo, uint8_t* kind) {
    int k = 0;
    for (u64 m = find_correct_moves(own, enemy); m; m &= m - 1, ++k) {
        const int sq = ctz64(m);
        u64 co, ce, hi, lo;
        const bool kept = child(own, enemy, sq, co, ce);
        canonical(co, ce, hi, lo);
        square[k] = (uint8_t)sq;
        c_own[k] = co;
        c_enemy[k] = ce;
        c_hi[k] = hi;
        c_lo[k] = lo;
        kind[k] = kept ? kChildKept : find_correct_moves(ce, co) ? kChildPass : kChildOver;
        child_index[k] = kept ? find_key(next_hi, next_lo, n_next, hi, lo) : -1;
    }
    return k;
}

}  // namespace openings
}  // namespace rz
