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
//
// Transposition table: whatever a frame proves ("value(own, enemy) >= t" is TRUE or FALSE) is a fact about the game,
// independent of the probe, the root, the call and the time slice.  So every lane of every probe shares one table of
// proven bounds lo <= value <= hi per position; a frame entered with t <= lo or t > hi is decided without search, and a
// stored best-move hint is tried first otherwise.  Only proven facts are stored, and the booleans do not depend on the
// move order, so the table changes the work, never an answer.
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
    int8_t cur;             // the move being explored (the proving move once the frame is decided TRUE)
    int8_t hint;            // the table's move, tried before the move order; -1 none
    int8_t pad[4];
};
static_assert(sizeof(LeafFrame) == 32, "leaf frame layout");

// ------------------------------------------------------------------------------------------------------- probe forests
//
// A probe forest (rz_solver_deep.cu) is a node table whose roots are the probes' questions.  The kernel and the host's
// copy of the tree ask roots_answered() whether the forest can end.

enum : int32_t { kOpen = 0, kTrue = 1, kFalse = 2 };

// `flip` of a root holds the forest's question: 0 or 1, the lowest root whose answer is that value (or all decided); or
// kEveryRoot, every root decided.
constexpr int kEveryRoot = 2;

struct Node {  // 24 B, written by the host only
    u64 own, enemy;
    int32_t parent;  // -1: a root
    int8_t t;        // the question: value(own to move) >= t ?
    int8_t flip;     // 1: the node's answer is negated for its parent (opponent to move); 0: pass.  Roots: the question
    int8_t empties;
    int8_t leaf;
};

RZ_HD bool roots_answered(const volatile int32_t* status, const Node* nodes, int n_roots) {
    // the lowest root whose answer is the wanted one, with every lower root decided the other way; or all decided
    for (int i = 0; i < n_roots; ++i) {
        const int s = status[i];
        if (s == kOpen) return false;
        const int f = nodes[i].flip;
        if (f != kEveryRoot && (s == kTrue) == (f != 0)) return true;
    }
    return true;
}

// One round of rz_solve_deep_moves over n moves with bounds lo[k] <= value <= hi[k]: t[k] = the threshold its root asks
// ("does the move reach t?": 1, then 0, then the middle of its bounds), or kNoProbe when the move is exact or, with
// n_best > 0, its hi is below the n_best-th largest lo (it cannot be among the best n_best).  Returns the open moves.
constexpr int kNoProbe = -128;
constexpr int kMaxMoveRounds = 8;  // t = 1, t = 0 and six halvings narrow [-64, 64] to one value
RZ_HD int plan_round(const int* lo, const int* hi, int n, int n_best, int* t) {
    int cut = -65;
    if (n_best > 0 && n_best <= n)
        for (int k = 0; k < n; ++k) {  // the n_best-th largest lo: the largest lo with n_best values at least as large
            int at_least = 0;
            for (int j = 0; j < n; ++j) at_least += lo[j] >= lo[k];
            if (at_least >= n_best && lo[k] > cut) cut = lo[k];
        }
    int open = 0;
    for (int k = 0; k < n; ++k) {
        const int l = lo[k], h = hi[k];
        t[k] = l >= h || h < cut ? kNoProbe : l <= 0 && h >= 1 ? 1 : l <= -1 && h >= 0 ? 0 : l + (h - l + 1) / 2;
        open += t[k] != kNoProbe;
    }
    return open;
}

// ------------------------------------------------------------------------------------------------ transposition table
//
// An HBM array of buckets of kTableWays entries (one 128-byte line), indexed by the lane solver's position hash.  An
// entry holds the full position, so a hash collision is a miss, never a wrong bound.  Concurrency is the evaluation
// cache's sequence protocol (rz_eval_cache.cuh): a writer claims an entry by a CAS of its sequence word to odd, writes,
// and publishes the next even value; a reader takes an entry only when it saw the same even word before and after
// copying it, with the right key.  A writer that loses the race drops its store and a reader that loses it sees a
// miss: both cost work, never correctness.  A store merges into the position's entry (bounds only tighten) or replaces
// the bucket's entry with the fewest empties.  (0, 0) is never a position with a legal move: it marks an empty entry.

constexpr int kTableWays = 4;
// Frames with fewer empties are neither looked up nor stored: their subtrees cost less to search than the lookup
// (DESIGN.md section 5 has the measurement behind the value).
#ifndef RZ_DEEP_TABLE_MIN_EMPTIES
#define RZ_DEEP_TABLE_MIN_EMPTIES 6
#endif
constexpr int kTableMinEmpties = RZ_DEEP_TABLE_MIN_EMPTIES;

struct __align__(32) TableEntry {  // 32 B
    u64 own, enemy;  // the position, own to move; (0, 0): empty
    uint32_t seq;    // odd while a writer holds the entry
    int8_t lo, hi;   // proven bounds on the exact final disc difference for own (empties not awarded); unknown: -64, 64
    int8_t move;     // the move that proved the last TRUE answer, -1 none
    int8_t empties;
    uint32_t pad[2];
};
static_assert(sizeof(TableEntry) == 32, "table entry layout");

struct Table {
    TableEntry* entries;  // [mask + 1][kTableWays]
    u64 mask;             // buckets - 1 (a power of two)
};

// Per-lane event counts (rz_deep_table_stats), summed into the workspace at the end of a slice.
enum { kTabLookups, kTabCutoffs, kTabHints, kTabStores, kTabReplaced, kTabMerges, kTabDropped, kTabCounters };

template <class T>
RZ_HD T load_cg(const T* p) {  // past the (incoherent) L1: another SM may have written the line
#ifdef __CUDA_ARCH__
    return __ldcg(p);
#else
    return *p;
#endif
}
RZ_HD uint32_t load_seq(const uint32_t* p) { return *(const volatile uint32_t*)p; }
RZ_HD bool claim_seq(uint32_t* p, uint32_t s) {
#ifdef __CUDA_ARCH__
    return atomicCAS(p, s, s + 1u) == s;
#else
    if (*p != s) return false;
    *p = s + 1u;
    return true;
#endif
}
RZ_HD void publish_seq(uint32_t* p, uint32_t s) {
#ifdef __CUDA_ARCH__
    atomicExch(p, s);
#else
    *p = s;
#endif
}

RZ_HD TableEntry* table_bucket(const Table& tab, u64 own, u64 enemy) {
    return tab.entries + (size_t)(solver::TT::mix(own, enemy) & tab.mask) * kTableWays;
}

// A consistent copy of the entry of (own, enemy): false when the position is absent or a writer held its entry.
RZ_HD bool table_lookup(const Table& tab, u64 own, u64 enemy, int& lo, int& hi, int& move) {
    TableEntry* b = table_bucket(tab, own, enemy);
    for (int w = 0; w < kTableWays; ++w) {
        TableEntry* e = b + w;
        if (load_cg(&e->own) != own || load_cg(&e->enemy) != enemy) continue;
        const uint32_t s1 = load_seq(&e->seq);
        solver::publish_fence();
        const u64 o = load_cg(&e->own), en = load_cg(&e->enemy);
        const uint32_t v = load_cg(reinterpret_cast<const uint32_t*>(&e->lo));
        solver::publish_fence();
        const uint32_t s2 = load_seq(&e->seq);
        if (s1 != s2 || (s1 & 1u) || o != own || en != enemy) return false;
        lo = (int8_t)(v & 0xFF); hi = (int8_t)(v >> 8 & 0xFF); move = (int8_t)(v >> 16 & 0xFF);
        return true;
    }
    return false;
}

// Record the proven bounds lo <= value(own, enemy) <= hi (and the proving move, or -1).  cnt: kTabCounters counts.
RZ_HD void table_store(const Table& tab, u64 own, u64 enemy, int empties, int lo, int hi, int move, uint32_t* cnt) {
    TableEntry* b = table_bucket(tab, own, enemy);
    int way = 0, least = 99;
    for (int w = 0; w < kTableWays; ++w) {
        const TableEntry* e = b + w;
        if (load_cg(&e->own) == own && load_cg(&e->enemy) == enemy) { way = w; break; }
        const int em = load_cg(reinterpret_cast<const uint32_t*>(&e->lo)) >> 24;
        if (em < least) { least = em; way = w; }
    }
    TableEntry* e = b + way;
    const uint32_t s = load_seq(&e->seq);
    if ((s & 1u) || !claim_seq(&e->seq, s)) { ++cnt[kTabDropped]; return; }  // another writer holds the entry
    solver::publish_fence();
    const u64 o = load_cg(&e->own), en = load_cg(&e->enemy);
    if (o == own && en == enemy) {  // merge under the claim: bounds only tighten
        const uint32_t v = load_cg(reinterpret_cast<const uint32_t*>(&e->lo));
        const int lo0 = (int8_t)(v & 0xFF), hi0 = (int8_t)(v >> 8 & 0xFF);
        if (lo0 > lo) lo = lo0;
        if (hi0 < hi) hi = hi0;
        if (move < 0) move = (int8_t)(v >> 16 & 0xFF);
        ++cnt[kTabMerges];
    } else {
        if (o | en) ++cnt[kTabReplaced];
        e->own = own; e->enemy = enemy; e->empties = (int8_t)empties;
        ++cnt[kTabStores];
    }
    e->lo = (int8_t)lo; e->hi = (int8_t)hi; e->move = (int8_t)move;
    solver::publish_fence();
    publish_seq(&e->seq, s + 2u);
}

// What the leaf machine asks of a table: enter(C) for a frame about to be searched returns 1 / 0 when a stored bound
// decides it (and sets C.hint otherwise, returning -1); decided(F, r) records a frame's answer.
struct NoTable {
    RZ_HD int enter(LeafFrame&) { return -1; }
    RZ_HD void decided(const LeafFrame&, bool) {}
};

struct TableLane {  // one lane's use of the table, with its own counts
    Table tab;
    uint32_t cnt[kTabCounters];

    RZ_HD int enter(LeafFrame& C) {
        if (64 - popc64(C.own | C.enemy) < kTableMinEmpties) return -1;
        ++cnt[kTabLookups];
        int lo, hi, move;
        if (!table_lookup(tab, C.own, C.enemy, lo, hi, move)) return -1;
        if (lo >= C.t || hi < C.t) { ++cnt[kTabCutoffs]; return lo >= C.t; }
        if (move >= 0 && (C.moves >> move & 1)) { C.hint = (int8_t)move; ++cnt[kTabHints]; }
        return -1;
    }
    RZ_HD void decided(const LeafFrame& F, bool r) { store(F.own, F.enemy, F.t, r, r ? F.cur : -1); }
    // "value(own, enemy) >= t" is r; move: the move that proved it TRUE, or -1
    RZ_HD void store(u64 own, u64 enemy, int t, bool r, int move) {
        const int empties = 64 - popc64(own | enemy);
        if (empties < kTableMinEmpties) return;
        table_store(tab, own, enemy, empties, r ? t : -64, r ? 64 : t - 1, move, cnt);
    }
};

// The child of (own, enemy) reached by the move at square a, seen from whoever moves next.  Returns false (and sets
// `diff`, the final disc difference for the side that played a) when the game is over after the move.
RZ_HD bool child_after(u64 own, u64 enemy, int a, int t, LeafFrame& c, int& diff) {
    const u64 fl = calc_flip(a, own, enemy);
    const u64 own2 = (own ^ fl) | (1ULL << a), en2 = enemy ^ fl;
    const u64 m = find_correct_moves(en2, own2);
    c.cur = c.hint = -1;
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
    F.cur = F.hint = -1;
    depth = 0;
}

// Advance the leaf whose stack is stk[0..depth] (stk[depth] = the frame being worked on).  Every `poll_every` node steps
// `keep_going()` is asked; when it says no the machine parks its working frame and returns kLeafSuspended.  Otherwise it
// runs to the answer of the root question.  `steps` is increased by the node steps made.  Each child frame is offered to
// `table.enter` before it is searched, and each decided frame to `table.decided` (the root frame's own lookup is the
// caller's, after leaf_init).
template <class Tab, class KeepGoing>
RZ_HD int leaf_advance(LeafFrame* stk, int& depth, long long& steps, int poll_every, Tab& table, KeepGoing&& keep_going) {
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
            const int a = F.hint >= 0 ? F.hint
                                      : solver::pick_move(F.own, F.enemy, F.moves, 64 - popc64(F.own | F.enemy) >= kOrderMinEmpties);
            F.hint = -1;
            F.moves &= ~(1ULL << a);
            F.cur = (int8_t)a;
            LeafFrame C;
            int diff;
            if (child_after(F.own, F.enemy, a, F.t, C, diff)) {
                const int known = table.enter(C);
                if (known < 0) {  // descend
                    stk[d++] = F;
                    F = C;
                    continue;
                }
                if (C.flip ? known : !known) continue;  // a stored bound says the child does not prove F
                r = true;
            } else {
                if (diff < F.t) continue;  // game over below the threshold: try the next move
                r = true;
            }
        }
        // F is decided (value >= F.t is r): hand it up until a frame is left that still has to try moves
        while (true) {
            table.decided(F, r);
            if (d == 0) { stk[0] = F; depth = 0; steps += n; return r ? kLeafTrue : kLeafFalse; }
            const bool proves_parent = F.flip ? !r : r;
            F = stk[--d];
            if (!proves_parent) break;
            r = true;
        }
    }
}

template <class KeepGoing>
RZ_HD int leaf_advance(LeafFrame* stk, int& depth, long long& steps, int poll_every, KeepGoing&& keep_going) {
    NoTable none;
    return leaf_advance(stk, depth, steps, poll_every, none, keep_going);
}

}  // namespace deep
}  // namespace rz
