// rz_openings.cuh -- one expansion step of the opening enumerator (rz_openings.cu), __host__ __device__ so that the
// host check (tests/support/openings_check.cu) runs the same code.
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

}  // namespace openings
}  // namespace rz
