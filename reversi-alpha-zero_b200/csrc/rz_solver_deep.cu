// rz_solver_deep.cu -- exact endgame solver that puts the whole device on one position (rz_solve_deep, include/rz_engine.h).
//
// The value is found by null-window probes "value >= t?" (t = 1, then 0, then bisection: at most 8 probes over
// [-64, 64]); the move by one more forest of probes over the root moves whose standing the value probes left open.
// One probe is an AND/OR tree:
//   * split: the host expands the probe root breadth-first in the lane solver's move order into a node table until the
//     frontier holds `leaf_target` leaves or every leaf is down to `leaf_floor` empties.  A move flips the threshold to
//     1 - t in the child's frame, a pass keeps side and threshold; finished games resolve when they are created;
//   * leaves: a persistent kernel runs in slices of `slice_us`; every lane claims leaves in depth-first move order and runs
//     the resumable null-window machine of rz_solver_deep.cuh on them, polling every kPollEvery node steps whether an
//     ancestor has been decided meanwhile (then the leaf is dropped) or the slice is over (then its stack is parked);
//   * resolution: a node is TRUE once one child proves it, FALSE once all children have failed to (a pending-children
//     counter); each decision is one CAS on the status word and climbs until it meets an ancestor already decided;
//   * between slices the host checks the timeout, and when fewer open leaves are left than lanes it re-splits the open
//     leaves that have run longest into their children (dropping their parked stacks), so skewed subtrees spread out;
//   * the transposition table (rz_solver_deep.cuh) is shared by every lane and kept across probes and calls: the leaf
//     machines look up the frames they enter and store the frames they decide, and resolve() stores the split-tree nodes
//     it decides, which are the largest subtrees and the first ones the next probe revisits.
// Booleans combine exactly, so the answer depends on nothing but the position (and on the timeout, only whether it hits).
//
// rz_solve_deep_moves asks the forest's other question, "every root decided": each round is one forest with one root per
// root move still open, each at its own threshold, so every move's value is narrowed at once (solve_moves).
#include <algorithm>
#include <chrono>
#include <vector>

#include "rz_common.cuh"
#include "rz_solver_deep.cuh"

namespace rz {
namespace deep {

constexpr int kBlockThreads = 128;
constexpr int kBlocksPerSm = 4;
constexpr int kPollEvery = 64;        // node steps between two abort / deadline checks of a leaf
constexpr int kMaxNodes = 1 << 21;    // node table capacity per probe
constexpr int kMaxRoots = 32;         // roots of a forest (one per root move)
constexpr int kDefaultSliceUs = 4000;
constexpr int kDefaultLeafFloor = 10;
constexpr int kCtxPerLane = 2;        // parked stacks per lane
constexpr long long kDefaultTableBytes = 1LL << 30;

struct SliceArgs {
    const Node* nodes;
    int32_t* status;
    int32_t* pending;
    int32_t* ctx;              // parked stack of a leaf: slot index, -1 none
    unsigned long long* steps; // node steps a leaf has run
    const int32_t* claim;      // open leaves in depth-first order
    int32_t n_claim;
    int32_t* claim_next;
    int32_t* stop;             // set when the roots answer the question
    int32_t n_roots;
    LeafFrame* ctx_frames;     // kLeafStack frames per slot
    int32_t* ctx_depth;
    const int32_t* free_slots;
    int32_t n_free;
    int32_t* free_next;
    unsigned long long* total_steps;
    long long slice_ns;
    Table table;
    unsigned long long* table_counts;  // kTabCounters
};

__device__ bool decided_above(const SliceArgs& a, int node) {
    const volatile int32_t* st = a.status;
    if (*(volatile int32_t*)a.stop) return true;
    for (int c = node; c >= 0; c = a.nodes[c].parent)
        if (st[c] != kOpen) return true;
    return false;
}

// The leaf `node` is decided r: climb while it decides ancestors, storing each ancestor it decides in the table (the
// leaf's own answer is stored by its machine, or came from the table).
__device__ void resolve(const SliceArgs& a, int node, bool r, TableLane& tl) {
    int c = node, from = -1;  // from: the child whose answer decided c
    while (true) {
        if (atomicCAS(&a.status[c], kOpen, r ? kTrue : kFalse) != kOpen) return;
        const Node& n = a.nodes[c];
        if (from >= 0) {  // TRUE: the proving move is the square the child has and c has not
            const u64 placed = (a.nodes[from].own | a.nodes[from].enemy) & ~(n.own | n.enemy);
            tl.store(n.own, n.enemy, n.t, r, r && placed ? ctz64(placed) : -1);
        }
        const int p = n.parent;
        if (p < 0) {
            __threadfence();
            if (roots_answered(a.status, a.nodes, a.n_roots)) atomicExch(a.stop, 1);
            return;
        }
        if (n.flip ? !r : r) { r = true; from = c; c = p; continue; }
        if (atomicSub(&a.pending[p], 1) == 1) { r = false; from = c; c = p; continue; }
        return;
    }
}

__global__ void __launch_bounds__(kBlockThreads, kBlocksPerSm) deep_slice_kernel(SliceArgs a) {
    LeafFrame stk[kLeafStack];
    const long long deadline = solver::global_ns() + a.slice_ns;
    unsigned long long lane_steps = 0;
    TableLane tl;
    tl.tab = a.table;
    for (int k = 0; k < kTabCounters; ++k) tl.cnt[k] = 0;
    while (true) {
        if (*(volatile int32_t*)a.stop || solver::global_ns() > deadline) break;
        const int i = atomicAdd(a.claim_next, 1);
        if (i >= a.n_claim) break;
        const int node = a.claim[i];
        if (decided_above(a, node)) continue;
        int depth;
        const int slot = a.ctx[node];
        if (slot >= 0) {
            depth = a.ctx_depth[slot];
            const LeafFrame* src = a.ctx_frames + (size_t)slot * kLeafStack;
            for (int k = 0; k <= depth; ++k) stk[k] = src[k];
        } else {
            leaf_init(stk, depth, a.nodes[node].own, a.nodes[node].enemy, a.nodes[node].t);
            const int known = tl.enter(stk[0]);  // a stored bound may decide the leaf at once
            if (known >= 0) { resolve(a, node, known != 0, tl); continue; }
        }
        long long steps = 0;
        bool out_of_time = false;
        const int r = leaf_advance(stk, depth, steps, kPollEvery, tl, [&]() {
            if (decided_above(a, node)) return false;
            out_of_time = solver::global_ns() > deadline;
            return !out_of_time;
        });
        atomicAdd(&a.steps[node], (unsigned long long)steps);
        lane_steps += steps;
        if (r != kLeafSuspended) { resolve(a, node, r == kLeafTrue, tl); continue; }
        if (!out_of_time) continue;  // an ancestor was decided: the leaf is moot
        int s = slot;
        if (s < 0) {
            const int f = atomicAdd(a.free_next, 1);
            s = f < a.n_free ? a.free_slots[f] : -1;
        }
        if (s >= 0) {  // park the stack; without a free slot the leaf starts over in a later slice
            LeafFrame* dst = a.ctx_frames + (size_t)s * kLeafStack;
            for (int k = 0; k <= depth; ++k) dst[k] = stk[k];
            a.ctx_depth[s] = depth;
        }
        a.ctx[node] = s;
        break;
    }
    atomicAdd(a.total_steps, lane_steps);
    for (int k = 0; k < kTabCounters; ++k) {  // every lane of the grid's full warps gets here
        const unsigned v = __reduce_add_sync(0xffffffffu, tl.cnt[k]);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(a.table_counts + k, (unsigned long long)v);
    }
}

// Occupied entries of the table into *out.
__global__ void table_count_kernel(const TableEntry* e, size_t n, unsigned long long* out) {
    unsigned c = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        c += (e[i].own | e[i].enemy) != 0;
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

// ---------------------------------------------------------------------------------------------------------------- host

struct Tuning {
    int slice_us = 0, leaf_target = 0, leaf_floor = 0;  // 0: default
    long long table_bytes = 0;
    int generation = 0;  // counts the calls of rz_solve_deep_tune / rz_solve_deep_table
};
static Tuning g_tuning;

struct Workspace {
    int lanes = 0, ctx_slots = 0;
    Node* nodes = nullptr;
    int32_t *status = nullptr, *pending = nullptr, *ctx = nullptr, *claim = nullptr, *ctx_depth = nullptr, *free_slots = nullptr;
    int32_t* counters = nullptr;  // claim_next, stop, free_next, pad
    unsigned long long *steps = nullptr, *total_steps = nullptr;
    LeafFrame* ctx_frames = nullptr;
    Table table{nullptr, 0};
    size_t table_entries = 0;
    int table_generation = -1;  // the tuning the table was emptied for
    unsigned long long* table_counts = nullptr;  // kTabCounters, then the occupied count of rz_solve_deep_table_stats
};

// One probe forest on the host: the authoritative copy between slices.
struct Tree {
    std::vector<Node> nodes;
    std::vector<int32_t> status, pending, ctx, first_child, n_children;
    std::vector<unsigned long long> steps;
    int n_roots = 0;
    long long leaves = 0;

    int add(u64 own, u64 enemy, int parent, int t, int flip) {
        Node n;
        n.own = own; n.enemy = enemy; n.parent = parent; n.t = (int8_t)t; n.flip = (int8_t)flip;
        n.empties = (int8_t)(64 - popc64(own | enemy)); n.leaf = 1;
        nodes.push_back(n);
        status.push_back(kOpen); pending.push_back(0); ctx.push_back(-1); first_child.push_back(-1); n_children.push_back(0);
        steps.push_back(0);
        ++leaves;
        return (int)nodes.size() - 1;
    }
    bool decided_above(int c) const {
        for (; c >= 0; c = nodes[c].parent)
            if (status[c] != kOpen) return true;
        return false;
    }
    void resolve(int c, bool r) {  // resolve() of the kernel, sequential
        while (true) {
            if (status[c] != kOpen) return;
            status[c] = r ? kTrue : kFalse;
            const int p = nodes[c].parent;
            if (p < 0) return;
            if (nodes[c].flip ? !r : r) { r = true; c = p; continue; }
            if (--pending[p] == 0) { r = false; c = p; continue; }
            return;
        }
    }
    bool answered() const { return roots_answered(status.data(), nodes.data(), n_roots); }
    // Replace leaf i by its children in the lane solver's move order; finished games resolve at once.
    void expand(int i) {
        const Node n = nodes[i];
        u64 moves = find_correct_moves(n.own, n.enemy);
        const bool ordered = n.empties >= kOrderMinEmpties;
        const int first = (int)nodes.size();
        int count = 0;
        int terminal_sq[32], terminal_r[32], n_terminal = 0;
        nodes[i].leaf = 0; ctx[i] = -1; --leaves;
        first_child[i] = first;
        while (moves) {
            const int a = solver::pick_move(n.own, n.enemy, moves, ordered);
            moves &= ~(1ULL << a);
            LeafFrame c;
            int diff;
            if (child_after(n.own, n.enemy, a, n.t, c, diff)) {
                add(c.own, c.enemy, i, c.t, c.flip);
            } else {  // game over: a node that is decided on creation (flip 0: its answer is the parent's)
                const int k = add(0, 0, i, 0, 0);
                nodes[k].leaf = 0; nodes[k].empties = 0; --leaves;
                terminal_sq[n_terminal] = k; terminal_r[n_terminal++] = diff >= n.t;
            }
            ++count;
        }
        n_children[i] = count;
        pending[i] = count;
        for (int k = 0; k < n_terminal; ++k) resolve(terminal_sq[k], terminal_r[k] != 0);
    }
    // open leaves (no decided ancestor), depth first in move order
    void open_leaves(std::vector<int32_t>& out) const {
        out.clear();
        std::vector<int> stack;
        for (int r = n_roots - 1; r >= 0; --r) stack.push_back(r);
        while (!stack.empty()) {
            const int c = stack.back();
            stack.pop_back();
            if (status[c] != kOpen) continue;
            if (nodes[c].leaf) { out.push_back(c); continue; }
            for (int k = n_children[c] - 1; k >= 0; --k) stack.push_back(first_child[c] + k);
        }
    }
};

struct ProbeRun {
    int slice_us, leaf_target, leaf_floor;
    std::chrono::steady_clock::time_point t0, deadline;
    const volatile int32_t* stop;  // the caller's stop flag (nullable): nonzero ends the call like a timeout
    rz_deep_solve_stats* stats;
    unsigned long long steps0;     // the workspace's node steps when the run began (with stats)
    bool expired() const { return (stop && *stop) || std::chrono::steady_clock::now() > deadline; }
};

static int upload_and_run(Workspace& w, Tree& T, const std::vector<int32_t>& claim, const std::vector<int32_t>& free_slots,
                          int slice_us) {
    const size_t n = T.nodes.size();
    RZ_CUDA_TRY(cudaMemcpy(w.nodes, T.nodes.data(), n * sizeof(Node), cudaMemcpyHostToDevice));
    RZ_CUDA_TRY(cudaMemcpy(w.status, T.status.data(), n * 4, cudaMemcpyHostToDevice));
    RZ_CUDA_TRY(cudaMemcpy(w.pending, T.pending.data(), n * 4, cudaMemcpyHostToDevice));
    RZ_CUDA_TRY(cudaMemcpy(w.ctx, T.ctx.data(), n * 4, cudaMemcpyHostToDevice));
    RZ_CUDA_TRY(cudaMemcpy(w.steps, T.steps.data(), n * 8, cudaMemcpyHostToDevice));
    RZ_CUDA_TRY(cudaMemcpy(w.claim, claim.data(), claim.size() * 4, cudaMemcpyHostToDevice));
    if (!free_slots.empty())
        RZ_CUDA_TRY(cudaMemcpy(w.free_slots, free_slots.data(), free_slots.size() * 4, cudaMemcpyHostToDevice));
    RZ_CUDA_TRY(cudaMemset(w.counters, 0, 4 * sizeof(int32_t)));
    SliceArgs a;
    a.nodes = w.nodes; a.status = w.status; a.pending = w.pending; a.ctx = w.ctx; a.steps = w.steps;
    a.claim = w.claim; a.n_claim = (int32_t)claim.size(); a.claim_next = w.counters; a.stop = w.counters + 1;
    a.n_roots = T.n_roots; a.ctx_frames = w.ctx_frames; a.ctx_depth = w.ctx_depth;
    a.free_slots = w.free_slots; a.n_free = (int32_t)free_slots.size(); a.free_next = w.counters + 2;
    a.total_steps = w.total_steps; a.slice_ns = (long long)slice_us * 1000;
    a.table = w.table; a.table_counts = w.table_counts;
    deep_slice_kernel<<<(unsigned)(w.lanes / kBlockThreads), kBlockThreads>>>(a);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaMemcpy(T.status.data(), w.status, n * 4, cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(T.pending.data(), w.pending, n * 4, cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(T.ctx.data(), w.ctx, n * 4, cudaMemcpyDeviceToHost));
    RZ_CUDA_TRY(cudaMemcpy(T.steps.data(), w.steps, n * 8, cudaMemcpyDeviceToHost));
    return RZ_OK;
}

// Decide the roots of T as far as the forest's question needs.  *timed_out is set when the deadline passed, or the stop flag
// was raised, first.
static int run_forest(Workspace& w, Tree& T, const ProbeRun& P, bool* timed_out) {
    *timed_out = false;
    // split breadth-first, one level at a time, down to the leaf target or the leaf floor
    std::vector<int32_t> level, claim, free_slots;
    T.open_leaves(level);
    while (!T.answered() && T.leaves < P.leaf_target) {
        if (P.expired()) { *timed_out = true; return RZ_OK; }
        bool grew = false;
        for (int c : level) {
            if (T.leaves >= P.leaf_target || T.nodes.size() + 64 > (size_t)kMaxNodes) break;
            if (T.decided_above(c) || T.nodes[c].empties <= P.leaf_floor) continue;
            T.expand(c);
            grew = true;
        }
        if (!grew) break;
        T.open_leaves(level);
    }
    std::vector<int> order;
    std::vector<char> used(w.ctx_slots);
    while (!T.answered()) {
        if (P.expired()) { *timed_out = true; return RZ_OK; }
        T.open_leaves(claim);
        if ((int)claim.size() < w.lanes) {  // lanes would sit idle: re-split the longest-running open leaves
            order.clear();
            for (int c : claim)
                if (T.nodes[c].empties > P.leaf_floor && T.steps[c] > 0) order.push_back(c);
            std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return T.steps[x] > T.steps[y]; });
            long long open = (long long)claim.size();
            int split = 0;
            for (int c : order) {
                if (open >= w.lanes || T.nodes.size() + 64 > (size_t)kMaxNodes) break;
                if (T.decided_above(c)) continue;
                const long long before = T.leaves;
                T.expand(c);
                open += T.leaves - before;
                ++split;
            }
            if (split) {
                if (P.stats) P.stats->resplits += split;
                if (T.answered()) break;
                T.open_leaves(claim);
            }
        }
        RZ_REQUIRE(!claim.empty(), "rz_solve_deep: undecided roots without an open leaf");
        std::fill(used.begin(), used.end(), 0);
        for (int c : claim)
            if (T.ctx[c] >= 0) used[T.ctx[c]] = 1;
        free_slots.clear();
        for (int s = 0; s < w.ctx_slots; ++s)
            if (!used[s]) free_slots.push_back(s);
        RZ_TRY(upload_and_run(w, T, claim, free_slots, P.slice_us));
        if (P.stats) P.stats->slices += 1;
    }
    return RZ_OK;
}

constexpr int kMaxDevices = 64;
static Workspace* g_ws[kMaxDevices] = {};

static int current_device(int* dev) {
    RZ_CUDA_TRY(cudaGetDevice(dev));
    RZ_REQUIRE(*dev >= 0 && *dev < kMaxDevices, "rz_solve_deep: device index out of range");
    return RZ_OK;
}

static int clear_table(Workspace& w) {
    RZ_CUDA_TRY(cudaMemset(w.table.entries, 0, w.table_entries * sizeof(TableEntry)));
    RZ_CUDA_TRY(cudaMemset(w.table_counts, 0, (kTabCounters + 1) * sizeof(unsigned long long)));
    return RZ_OK;
}

// After a tuning call, an empty table of the size rz_solve_deep_table asked for (the largest power of two of buckets that
// fits), so that a test or measurement under the new tuning searches instead of answering from earlier proofs.
static int prepare_table(Workspace& w) {
    if (w.table_generation == g_tuning.generation) return RZ_OK;
    const long long bytes = g_tuning.table_bytes ? g_tuning.table_bytes : kDefaultTableBytes;
    u64 buckets = 1;
    while ((long long)(buckets * 2 * kTableWays * sizeof(TableEntry)) <= bytes) buckets *= 2;
    if (!w.table.entries || w.table.mask + 1 != buckets) {
        if (w.table.entries) RZ_CUDA_TRY(cudaFree(w.table.entries));
        w.table.entries = nullptr;
        w.table_entries = (size_t)buckets * kTableWays;
        RZ_CUDA_TRY(cudaMalloc((void**)&w.table.entries, w.table_entries * sizeof(TableEntry)));
        w.table.mask = buckets - 1;
    }
    w.table_generation = g_tuning.generation;
    return clear_table(w);
}

static int workspace(Workspace** out) {
    int dev = 0;
    RZ_TRY(current_device(&dev));
    if (!g_ws[dev]) {
        Workspace* w = new Workspace;
        w->lanes = num_sms() * kBlocksPerSm * kBlockThreads;
        w->ctx_slots = w->lanes * kCtxPerLane;
        RZ_CUDA_TRY(cudaMalloc((void**)&w->nodes, (size_t)kMaxNodes * sizeof(Node)));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->status, (size_t)kMaxNodes * 4));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->pending, (size_t)kMaxNodes * 4));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->ctx, (size_t)kMaxNodes * 4));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->claim, (size_t)kMaxNodes * 4));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->steps, (size_t)kMaxNodes * 8));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->ctx_depth, (size_t)w->ctx_slots * 4));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->free_slots, (size_t)w->ctx_slots * 4));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->ctx_frames, (size_t)w->ctx_slots * kLeafStack * sizeof(LeafFrame)));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->counters, 4 * sizeof(int32_t)));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->total_steps, sizeof(unsigned long long)));
        RZ_CUDA_TRY(cudaMalloc((void**)&w->table_counts, (kTabCounters + 1) * sizeof(unsigned long long)));
        g_ws[dev] = w;
    }
    RZ_TRY(prepare_table(*g_ws[dev]));
    *out = g_ws[dev];
    return RZ_OK;
}

// One solve's run under the current tuning, from now until `timeout_s` has passed or *stop is set; end_run fills the
// node steps and seconds of its stats.
static int begin_run(const Workspace& w, double timeout_s, const volatile int32_t* stop, rz_deep_solve_stats* stats, ProbeRun& P) {
    P.t0 = std::chrono::steady_clock::now();
    P.slice_us = g_tuning.slice_us ? g_tuning.slice_us : kDefaultSliceUs;
    P.leaf_target = g_tuning.leaf_target ? g_tuning.leaf_target : w.lanes;
    P.leaf_floor = g_tuning.leaf_floor ? g_tuning.leaf_floor : kDefaultLeafFloor;
    P.deadline = P.t0 + std::chrono::duration_cast<std::chrono::steady_clock::duration>(std::chrono::duration<double>(timeout_s));
    P.stop = stop;
    P.stats = stats;
    P.steps0 = 0;
    if (stats) RZ_CUDA_TRY(cudaMemcpy(&P.steps0, w.total_steps, 8, cudaMemcpyDeviceToHost));
    return RZ_OK;
}

static int end_run(const Workspace& w, const ProbeRun& P) {
    if (!P.stats) return RZ_OK;
    unsigned long long steps1 = 0;
    RZ_CUDA_TRY(cudaMemcpy(&steps1, w.total_steps, 8, cudaMemcpyDeviceToHost));
    P.stats->node_steps = (int64_t)(steps1 - P.steps0);
    P.stats->seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - P.t0).count();
    return RZ_OK;
}

// Bounds on the value of each root move, in the root mover's frame, learned from decided root children.
struct MoveBounds {
    int lo[64], hi[64];
};

static void learn_root_children(const Tree& T, int root, MoveBounds& B, const int* child_sq) {
    if (T.first_child[root] < 0) return;
    for (int k = 0; k < T.n_children[root]; ++k) {
        const int c = T.first_child[root] + k;
        const int s = T.status[c];
        if (s == kOpen) continue;
        const int sq = child_sq[k];
        // the child's answer r to "value_c >= t_c"; flip: the move's value is -value_c, else value_c
        const Node& n = T.nodes[c];
        const bool r = s == kTrue;
        if (n.empties == 0 && !n.leaf && n.own == 0 && n.enemy == 0) continue;  // a finished game: known exactly already
        if (n.flip) {
            if (r) B.hi[sq] = std::min(B.hi[sq], -n.t); else B.lo[sq] = std::max(B.lo[sq], 1 - n.t);
        } else {
            if (r) B.lo[sq] = std::max(B.lo[sq], (int)n.t); else B.hi[sq] = std::min(B.hi[sq], n.t - 1);
        }
    }
}

// The root moves of (own, enemy) in the split's order into child_sq; bounds [-64, 64], exact where the move ends the game.
static int root_moves(u64 own, u64 enemy, u64 legal, int* child_sq, MoveBounds& B) {
    int n_moves = 0;
    for (int s = 0; s < 64; ++s) { B.lo[s] = -64; B.hi[s] = 64; }
    const bool ordered = 64 - popc64(own | enemy) >= kOrderMinEmpties;
    while (legal) {
        const int a = solver::pick_move(own, enemy, legal, ordered);
        legal &= ~(1ULL << a);
        child_sq[n_moves++] = a;
        LeafFrame c;
        int diff;
        if (!child_after(own, enemy, a, 0, c, diff)) B.lo[a] = B.hi[a] = diff;
    }
    return n_moves;
}

static int solve_one(Workspace& w, u64 own, u64 enemy, int8_t* move_out, int8_t* score_out, const ProbeRun& P) {
    *move_out = -1; *score_out = 0;
    const u64 legal = find_correct_moves(own, enemy);
    if (!legal || 64 - popc64(own | enemy) > kDeepMaxEmpties) return RZ_OK;
    // root moves in the split's order, and their exact values where the game ends
    int child_sq[kMaxRoots];
    MoveBounds B;
    root_moves(own, enemy, legal, child_sq, B);
    Tree T;
    bool timed_out = false;
    auto probe = [&](int t, bool* r) -> int {
        T = Tree();
        T.n_roots = 1;
        T.add(own, enemy, -1, t, 0);
        if (P.stats) P.stats->probes += 1;
        RZ_TRY(run_forest(w, T, P, &timed_out));
        if (P.stats) P.stats->leaves += T.leaves;
        *r = T.status[0] == kTrue;
        learn_root_children(T, 0, B, child_sq);
        return RZ_OK;
    };
    // value: t = 1, t = 0, then bisection inside the known sign range
    int lo = -64, hi = 64;
    bool r;
    RZ_TRY(probe(1, &r));
    if (timed_out) return RZ_OK;
    if (r) lo = 1; else hi = 0;
    if (!r) {
        RZ_TRY(probe(0, &r));
        if (timed_out) return RZ_OK;
        if (r) lo = 0; else hi = -1;
    }
    while (lo < hi) {
        const int mid = lo + (hi - lo + 1) / 2;
        RZ_TRY(probe(mid, &r));
        if (timed_out) return RZ_OK;
        if (r) lo = mid; else hi = mid - 1;
    }
    const int v = lo;
    // move: the first square whose move reaches v.  Squares already known to fall short are skipped; the open ones below
    // the first known best move are probed together, one root each ("does this move reach v?")
    int known_best = 64;
    for (int s = 0; s < 64; ++s)
        if ((legal >> s & 1) && B.lo[s] >= v) { known_best = s; break; }
    int open_sq[kMaxRoots], n_open = 0;
    for (int s = 0; s < known_best; ++s)
        if ((legal >> s & 1) && B.hi[s] >= v) open_sq[n_open++] = s;
    int best = known_best;
    if (n_open) {
        T = Tree();
        for (int k = 0; k < n_open; ++k) {
            LeafFrame c;
            int diff;
            child_after(own, enemy, open_sq[k], v, c, diff);  // never a finished game: those are known exactly
            // opponent to move: the move reaches v iff NOT (value_c >= 1 - v); pass: iff value_c >= v.  `flip` of a
            // root holds the wanted answer.
            T.add(c.own, c.enemy, -1, c.t, c.flip ? 0 : 1);
        }
        T.n_roots = n_open;
        if (P.stats) P.stats->probes += 1;
        RZ_TRY(run_forest(w, T, P, &timed_out));
        if (timed_out) return RZ_OK;
        if (P.stats) P.stats->leaves += T.leaves;
        for (int k = 0; k < n_open; ++k)
            if ((T.status[k] == kTrue) == (T.nodes[k].flip != 0)) { best = open_sq[k]; break; }
    }
    if (best >= 64) return RZ_OK;  // cannot happen: some move reaches the value
    *move_out = (int8_t)best; *score_out = (int8_t)v;
    return RZ_OK;
}

// Bounds B.lo <= value <= B.hi of every legal root move of (own, enemy), in the root mover's frame (rz_solve_deep_moves).
// Each round is one forest with one root per open move, asking "does this move reach t?" at the move's own t (1, then
// 0, then the middle of its bounds), and runs until every root is decided.  A move is open while it is inexact and, with
// n_best > 0, its hi is not below the n_best-th largest lo.  lo / hi receive the bounds after every round, and on_round
// (nullable) sees them.  On a timeout or stop the bounds proven so far stay, and they always hold.  The plan of each
// round is plan_round (rz_solver_deep.cuh).
static int solve_moves(Workspace& w, u64 own, u64 enemy, u64 legal, int n_best, int8_t* lo, int8_t* hi,
                       rz_deep_moves_cb on_round, void* user, const ProbeRun& P) {
    int child_sq[kMaxRoots];
    MoveBounds B;
    const int n_moves = root_moves(own, enemy, legal, child_sq, B);
    auto publish = [&] {
        for (int k = 0; k < n_moves; ++k) { lo[child_sq[k]] = (int8_t)B.lo[child_sq[k]]; hi[child_sq[k]] = (int8_t)B.hi[child_sq[k]]; }
    };
    publish();
    Tree T;
    for (int round = 0; round < kMaxMoveRounds; ++round) {
        int lo_k[kMaxRoots], hi_k[kMaxRoots], t_k[kMaxRoots];
        for (int k = 0; k < n_moves; ++k) { lo_k[k] = B.lo[child_sq[k]]; hi_k[k] = B.hi[child_sq[k]]; }
        plan_round(lo_k, hi_k, n_moves, n_best, t_k);
        int open_sq[kMaxRoots], t_of[kMaxRoots], n_open = 0;
        bool pass_of[kMaxRoots];
        T = Tree();
        for (int k = 0; k < n_moves; ++k) {
            if (t_k[k] == kNoProbe) continue;
            const int s = child_sq[k], t = t_k[k];
            LeafFrame c;
            int diff;
            child_after(own, enemy, s, t, c, diff);  // never a finished game: those are exact already
            T.add(c.own, c.enemy, -1, c.t, kEveryRoot);
            open_sq[n_open] = s; t_of[n_open] = t; pass_of[n_open++] = c.flip == 0;
        }
        if (!n_open) break;
        T.n_roots = n_open;
        if (P.stats) P.stats->probes += 1;
        bool timed_out = false;
        RZ_TRY(run_forest(w, T, P, &timed_out));
        if (P.stats) P.stats->leaves += T.leaves;
        // opponent to move: the move reaches t iff NOT (value_c >= 1 - t); pass: iff value_c >= t.  A root left open by a
        // timeout proves nothing.
        for (int k = 0; k < n_open; ++k) {
            if (T.status[k] == kOpen) continue;
            const int s = open_sq[k];
            if ((T.status[k] == kTrue) == pass_of[k]) B.lo[s] = std::max(B.lo[s], t_of[k]);
            else B.hi[s] = std::min(B.hi[s], t_of[k] - 1);
        }
        publish();
        if (on_round) on_round(lo, hi, user);
        if (timed_out) break;
    }
    return RZ_OK;
}

}  // namespace deep
}  // namespace rz

using namespace rz;

extern "C" {

int rz_solve_deep_tune(int slice_us, int leaf_target, int leaf_floor) {
    RZ_REQUIRE(slice_us >= 0 && leaf_target >= 0 && leaf_floor >= 0, "rz_solve_deep_tune: negative argument");
    deep::g_tuning.slice_us = slice_us;
    deep::g_tuning.leaf_target = leaf_target;
    deep::g_tuning.leaf_floor = leaf_floor;
    ++deep::g_tuning.generation;
    return RZ_OK;
}

int rz_solve_deep_table(int64_t bytes) {
    RZ_REQUIRE(bytes >= 0, "rz_solve_deep_table: negative size");
    deep::g_tuning.table_bytes = bytes;
    ++deep::g_tuning.generation;
    return RZ_OK;
}

int rz_solve_deep_clear(void) {
    int dev = 0;
    RZ_TRY(deep::current_device(&dev));
    if (deep::g_ws[dev]) RZ_TRY(deep::clear_table(*deep::g_ws[dev]));
    return RZ_OK;
}

int rz_solve_deep_table_stats(rz_deep_table_stats* out) {
    RZ_REQUIRE(out, "rz_solve_deep_table_stats: null pointer");
    *out = rz_deep_table_stats{};
    int dev = 0;
    RZ_TRY(deep::current_device(&dev));
    deep::Workspace* w = deep::g_ws[dev];
    if (!w) return RZ_OK;
    unsigned long long* occupied = w->table_counts + deep::kTabCounters;
    RZ_CUDA_TRY(cudaMemset(occupied, 0, sizeof(unsigned long long)));
    deep::table_count_kernel<<<(unsigned)num_sms() * 8, 256>>>(w->table.entries, w->table_entries, occupied);
    RZ_LAUNCH_CHECK();
    unsigned long long c[deep::kTabCounters + 1];
    RZ_CUDA_TRY(cudaMemcpy(c, w->table_counts, sizeof(c), cudaMemcpyDeviceToHost));
    out->lookups = (int64_t)c[deep::kTabLookups];
    out->cutoffs = (int64_t)c[deep::kTabCutoffs];
    out->hints = (int64_t)c[deep::kTabHints];
    out->stores = (int64_t)c[deep::kTabStores];
    out->replaced = (int64_t)c[deep::kTabReplaced];
    out->merges = (int64_t)c[deep::kTabMerges];
    out->dropped = (int64_t)c[deep::kTabDropped];
    out->occupied = (int64_t)c[deep::kTabCounters];
    out->bytes = (int64_t)(w->table_entries * sizeof(deep::TableEntry));
    return RZ_OK;
}

int rz_solve_deep_with_stop(const uint64_t* own, const uint64_t* enemy, int8_t* move, int8_t* score, size_t n, double timeout_s,
                            const volatile int32_t* stop, rz_deep_solve_stats* stats) {
    RZ_REQUIRE(n == 0 || (own && enemy && move && score), "rz_solve_deep: null pointer");
    deep::Workspace* w = nullptr;
    if (n) RZ_TRY(deep::workspace(&w));
    for (size_t i = 0; i < n; ++i) {
        if (stats) stats[i] = rz_deep_solve_stats{};
        if (stop && *stop) { move[i] = -1; score[i] = 0; continue; }
        deep::ProbeRun P;
        RZ_TRY(deep::begin_run(*w, timeout_s, stop, stats ? stats + i : nullptr, P));
        RZ_TRY(deep::solve_one(*w, own[i], enemy[i], move + i, score + i, P));
        RZ_TRY(deep::end_run(*w, P));
    }
    return RZ_OK;
}

int rz_solve_deep_moves(uint64_t own, uint64_t enemy, int n_best, double timeout_s, const volatile int32_t* stop, int8_t* lo,
                        int8_t* hi, uint64_t* legal, rz_deep_moves_cb on_round, void* user, rz_deep_solve_stats* stats) {
    RZ_REQUIRE(lo && hi && legal, "rz_solve_deep_moves: null pointer");
    RZ_REQUIRE(n_best >= 0, "rz_solve_deep_moves: negative n_best");
    for (int s = 0; s < 64; ++s) lo[s] = hi[s] = 0;
    if (stats) *stats = rz_deep_solve_stats{};
    *legal = find_correct_moves(own, enemy);
    if (!*legal || 64 - popc64(own | enemy) > deep::kDeepMaxEmpties) { *legal = 0; return RZ_OK; }
    deep::Workspace* w = nullptr;
    RZ_TRY(deep::workspace(&w));
    deep::ProbeRun P;
    RZ_TRY(deep::begin_run(*w, timeout_s, stop, stats, P));
    RZ_TRY(deep::solve_moves(*w, own, enemy, *legal, n_best, lo, hi, on_round, user, P));
    return deep::end_run(*w, P);
}

int rz_solve_deep(const uint64_t* own, const uint64_t* enemy, int8_t* move, int8_t* score, size_t n, double timeout_s,
                  rz_deep_solve_stats* stats) {
    return rz_solve_deep_with_stop(own, enemy, move, score, n, timeout_s, nullptr, stats);
}

}  // extern "C"
