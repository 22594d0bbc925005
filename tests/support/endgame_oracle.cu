// Independent exact endgame oracle for the deep solver's tests: plain recursive negamax alpha-beta over rz_bitboard.cuh
// (with a table of proven bounds, keyed by the whole position, for speed), compiled for the HOST.  Reads lines "own enemy" (hex, the mover's frame) and prints "move score": the exact final disc
// difference (empties not awarded) and the FIRST square in ascending order that reaches it; "-1 0" when the mover has
// no legal move.  Shares nothing with the device solvers but the rules.
#include <cstdio>
#include <vector>
#include "rz_bitboard.cuh"
using namespace rz;

static long long g_nodes = 0;

// proven bounds lo <= value <= hi of positions with at least kTtMinEmpties empties, keyed by the whole position
struct Entry { u64 own, enemy; int lo, hi; };
constexpr int kTtBits = 22, kTtMinEmpties = 7;
static std::vector<Entry> g_tt(1u << kTtBits, Entry{0, 0, -65, 65});
static Entry& slot(u64 own, u64 enemy) {
    u64 h = own * 0x9E3779B97F4A7C15ULL ^ enemy * 0xC2B2AE3D27D4EB4FULL;
    return g_tt[(h ^ (h >> 29)) & ((1u << kTtBits) - 1)];
}

// exact value of (own to move) if it lies in (alpha, beta), else a bound on the side of the window it falls
static int negamax(u64 own, u64 enemy, int alpha, int beta, bool passed) {
    ++g_nodes;
    u64 moves = find_correct_moves(own, enemy);
    if (!moves) {
        if (passed) return popc64(own) - popc64(enemy);  // neither side can move: the game is over
        return -negamax(enemy, own, -beta, -alpha, true);
    }
    const bool cached = 64 - popc64(own | enemy) >= kTtMinEmpties;
    if (cached) {
        const Entry& e = slot(own, enemy);
        if (e.own == own && e.enemy == enemy) {
            if (e.lo >= beta) return e.lo;
            if (e.hi <= alpha) return e.hi;
            if (e.lo == e.hi) return e.lo;
            if (e.lo > alpha) alpha = e.lo;
            if (e.hi < beta) beta = e.hi;
        }
    }
    const int alpha0 = alpha;
    // children with the fewest opponent replies first: only speed, any order gives the same value
    int sq[32], mob[32], n = 0;
    const bool order = 64 - popc64(own | enemy) > 6;
    for (u64 m = moves; m; m &= m - 1) {
        const int a = ctz64(m);
        int k = n++;
        const int mb = order ? popc64(find_correct_moves(enemy ^ calc_flip(a, own, enemy), own | calc_flip(a, own, enemy) | (1ULL << a))) : 0;
        while (k > 0 && mob[k - 1] > mb) { sq[k] = sq[k - 1]; mob[k] = mob[k - 1]; --k; }
        sq[k] = a; mob[k] = mb;
    }
    int best = -65;
    for (int i = 0; i < n; ++i) {
        const u64 fl = calc_flip(sq[i], own, enemy);
        const int v = -negamax(enemy ^ fl, own | fl | (1ULL << sq[i]), -beta, -(alpha > best ? alpha : best), false);
        if (v > best) {
            best = v;
            if (best >= beta) break;
        }
    }
    if (cached) {
        Entry& e = slot(own, enemy);
        if (e.own != own || e.enemy != enemy) e = Entry{own, enemy, -65, 65};
        if (best <= alpha0) e.hi = best < e.hi ? best : e.hi;
        else if (best >= beta) e.lo = best > e.lo ? best : e.lo;
        else e.lo = e.hi = best;
    }
    return best;
}

int main() {
    unsigned long long own, enemy;
    while (scanf("%llx %llx", &own, &enemy) == 2) {
        const u64 moves = find_correct_moves(own, enemy);
        int move = -1, best = -65;
        // root: ascending squares; a later move replaces the best only if it is strictly better (window (best, 65))
        for (u64 m = moves; m; m &= m - 1) {
            const int a = ctz64(m);
            const u64 fl = calc_flip(a, own, enemy);
            const int v = -negamax(enemy ^ fl, own | fl | (1ULL << a), -65, -best, false);
            if (v > best) { best = v; move = a; }
        }
        printf("%d %d\n", move, move < 0 ? 0 : best);
        fflush(stdout);
    }
    fprintf(stderr, "nodes %lld\n", g_nodes);
    return 0;
}
