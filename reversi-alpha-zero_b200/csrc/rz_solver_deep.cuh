// rz_solver_deep.cuh -- the leaf machine of the whole-GPU exact endgame solver (rz_solver_deep.cu), __host__ __device__.
//
// A leaf answers one null-window question about a position: "is the exact final disc difference for the side to move
// (empties not awarded) >= t?".  Because the window (t - 1, t) has width one, every node is a boolean: a node is TRUE
// as soon as one move leads to a child that proves it (the child FALSE at 1 - t when the opponent replies, the child
// TRUE at the same t when the opponent has to pass), FALSE when no move does.  So a frame keeps no score, only its
// threshold and the moves it has not tried yet.
//
// The machine is an explicit stack, so a leaf can be advanced for a bounded number of node steps, parked in global
// memory and resumed by any lane later: the result never depends on where it was suspended.  Inner nodes try moves in
// the lane solver's order (rz_solver.cuh pick_move: the reply that leaves the opponent the fewest moves first).
#pragma once
#include "rz_solver.cuh"

namespace rz {
namespace deep {

constexpr int kDeepMaxEmpties = 30;  // larger positions are refused
// A frame is pushed per move and per forced pass, and two passes in a row end the game: depth <= 2 x empties.
constexpr int kLeafStack = 2 * kDeepMaxEmpties + 4;
constexpr int kOrderMinEmpties = solver::kOrderMinEmpties;

enum LeafResult { kLeafFalse = 0, kLeafTrue = 1, kLeafSuspended = 2 };

struct LeafFrame {  // 32 B
    u64 own, enemy, moves;  // position (side to move = own) and the moves not tried yet
    int8_t t;               // the question: value >= t ?
    int8_t flip;            // 1: the opponent moved into this frame (its answer is negated for the parent); 0: a pass
    int8_t pad[6];
};

// The child of (own, enemy) reached by the move at square a, seen from whoever moves next.  Returns false (and sets
// `diff`, the final disc difference for the side that played a) when the game is over after the move.
RZ_HD bool child_after(u64 own, u64 enemy, int a, int t, LeafFrame& c, int& diff) {
    const u64 fl = calc_flip(a, own, enemy);
    const u64 own2 = (own ^ fl) | (1ULL << a), en2 = enemy ^ fl;
    const u64 m = find_correct_moves(en2, own2);
    if (m) { c.own = en2; c.enemy = own2; c.moves = m; c.t = (int8_t)(1 - t); c.flip = 1; return true; }
    const u64 ms = find_correct_moves(own2, en2);
    if (ms) { c.own = own2; c.enemy = en2; c.moves = ms; c.t = (int8_t)t; c.flip = 0; return true; }
    diff = popc64(own2) - popc64(en2);
    return false;
}

// Stack root for the question "value(own, enemy) >= t"; the side to move must have a legal move.
RZ_HD void leaf_init(LeafFrame* stk, int& depth, u64 own, u64 enemy, int t) {
    LeafFrame& F = stk[0];
    F.own = own; F.enemy = enemy; F.moves = find_correct_moves(own, enemy); F.t = (int8_t)t; F.flip = 0;
    depth = 0;
}

// Advance the leaf whose stack is stk[0..depth] (stk[depth] = the frame being worked on).  Every `poll_every` node steps
// `keep_going()` is asked; when it says no the machine parks its working frame and returns kLeafSuspended.  Otherwise it
// runs to the answer of the root question.  `steps` is increased by the node steps made.
template <class KeepGoing>
RZ_HD int leaf_advance(LeafFrame* stk, int& depth, long long& steps, int poll_every, KeepGoing&& keep_going) {
    int d = depth;
    LeafFrame F = stk[d];
    int n = 0;
    while (true) {
        if (++n == poll_every) {
            steps += n; n = 0;
            if (!keep_going()) { stk[d] = F; depth = d; return kLeafSuspended; }
        }
        bool r;  // set when F is decided
        if (F.moves == 0) {
            r = false;
        } else {
            const int a = solver::pick_move(F.own, F.enemy, F.moves, 64 - popc64(F.own | F.enemy) >= kOrderMinEmpties);
            F.moves &= ~(1ULL << a);
            LeafFrame C;
            int diff;
            if (child_after(F.own, F.enemy, a, F.t, C, diff)) {  // descend
                stk[d++] = F;
                F = C;
                continue;
            }
            if (diff < F.t) continue;  // game over below the threshold: try the next move
            r = true;
        }
        // F is decided (value >= F.t is r): hand it up until a frame is left that still has to try moves
        while (true) {
            if (d == 0) { stk[0] = F; depth = 0; steps += n; return r ? kLeafTrue : kLeafFalse; }
            const bool proves_parent = F.flip ? !r : r;
            F = stk[--d];
            if (!proves_parent) break;
            r = true;
        }
    }
}

}  // namespace deep
}  // namespace rz
