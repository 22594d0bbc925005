// rz_engine.cu -- K2/K3/K6/K7: on-device MCTS self-play (agent/player.py ReversiPlayer,
// worker/self_play.py game loop) for thousands of concurrent games.
//
// Data layout (HBM, per game slot, flat arrays):
//   * transposition table: open-addressing hash (uint32 slots, generation-tagged so a new game needs no
//     clearing) -> node index; keys are (own, enemy) in the side-to-move's frame.  The reference keeps
//     statistics under CounterKey(black, white, next_player) and under the colour-swapped mirror key
//     with W negated (player.py:276-280,388-393): that is one table in the mover's frame (DESIGN.md).
//   * nodes (32 B): key, legal-move mask, first-edge index, per-player "expanded" bits
//     (each ReversiPlayer has its own `expanded` set even when statistics are shared, player.py:44-47).
//   * edges (16 B, legal moves only, ascending square order): visit count N, value sum W (fp32, mover's
//     frame), prior P already re-normalised over the legal moves (player.py:406-413).
//   * K descent slots (parallel_search_num) with the search path, K-entry pending / parked lists.
//   * two ply logs (double-buffered mailboxes) from which the host harvests finished games.
// One wave = one `tick` kernel (consume the previous evaluations: expand + backup; decide moves, step
// games, start new games; run up to K descents per game with virtual loss; gather the leaves with a
// warp-scan into one compact batch, already dihedral-transformed) + one network launch on the batch
// whose size the network kernel reads from device memory (no host round trip inside a wave).
// The arithmetic of selection / backup / move choice follows oracle/mcts.py operation by operation
// (fp32 priors and W, fp64 Q/U, numpy summation order), so that parity tests can demand exact equality.
// This translation unit is compiled with -fmad=false for that reason.
#include <deque>
#include <mutex>
#include <new>
#include <vector>
#include <stdlib.h>
#include <string.h>
#include "rz_bitboard.cuh"
#include "rz_net.cuh"
#include "rz_solver.cuh"

namespace rz {
namespace solver {
constexpr int kBlockThreads = 128;
// The engine's solver step: advance every unfinished request of a slot group for at most `budget_ns`, then queue what is
// still unfinished for the group's next wave.  `active` holds request-context indices: the unfinished ones of the last
// wave followed by those the tick kernel just added.  One CTA per SM.  A CTA of the tower kernel takes nearly all of an
// SM's registers, so these CTAs start only on SMs the other group's tower launch leaves free or after it ends; the budget
// bounds the time a CTA runs once it has started, not the stream time of the step.
__global__ void __launch_bounds__(kBlockThreads) solve_active_kernel(SolveCtx* __restrict__ ctx, const uint32_t* __restrict__ active,
                                                                     const uint32_t* __restrict__ n_active, uint32_t* __restrict__ next,
                                                                     uint32_t* __restrict__ n_next, u64* tt_base, long long budget_ns) {
    const uint32_t n = *n_active;
    if (n == 0) return;
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, total = gridDim.x * blockDim.x, n_warps = total >> 5;
    const long long deadline = global_ns() + budget_ns;
    const TT tt{tt_base + (size_t)tid * kTtEntries * kTtWordsPerEntry};
    // request r -> lane r / n_warps of warp r % n_warps: spreads a short list over all warps (few divergent lanes per warp)
    for (uint32_t r = (tid & 31u) * n_warps + (tid >> 5); r < n; r += total) {
        const uint32_t idx = active[r];
        if (!solve_advance(ctx + idx, tt, deadline)) next[atomicAdd(n_next, 1u)] = idx;
    }
}
}  // namespace solver

namespace eng {

// ---- Philox4x32-10 (same streams as oracle/philox.py) ------------------------------------------------
enum { P_DIHEDRAL = 0, P_MOVE = 1, P_NOISE = 2, P_GAME = 3 };

struct U4 { uint32_t x, y, z, w; };

__device__ __forceinline__ U4 philox(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    return U4{c0, c1, c2, c3};
}
__device__ __forceinline__ U4 draw(uint64_t seed, uint64_t game_id, uint32_t seq, uint32_t purpose, uint32_t idx) {
    return philox((uint32_t)game_id, seq, purpose, idx, (uint32_t)seed, (uint32_t)(seed >> 32));
}
__device__ __forceinline__ double u01(uint32_t x) { return ((double)x + 0.5) * (1.0 / 4294967296.0); }
__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
    return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

// ---- device-side structures ---------------------------------------------------------------------------
struct Node {  // 32 B
    u64 own, enemy, legal;
    uint32_t edge_base;
    uint8_t exp;   // bit (pid-1): expanded by that player
    uint8_t kpid;  // 0 in shared mode, else the player the table entry belongs to
    uint16_t pad;
};
struct __align__(16) Edge { int32_t n; float w; float p; int32_t pad; };

enum : uint8_t { D_FREE = 0, D_PENDING = 1, D_PARKED = 2 };
constexpr int kMaxK = 16;
constexpr int kMaxPath = 64;

struct Descent {
    u64 black, white;        // position reached so far
    u64 leaf_own, leaf_enemy;
    uint32_t leaf_index;     // row in the evaluation batch
    uint8_t next_player, status, dihedral, path_len;
    uint8_t leaf_mover_is_root;
    uint8_t kept;            // 1: the network result of this leaf was copied to keep_policy / keep_value
    uint8_t pad[2];
    uint32_t path[kMaxPath];  // edge index within the slot's arena | (mover_is_root << 31)
};

enum : uint8_t { PH_IDLE = 0, PH_SEARCH = 1, PH_DECIDE = 2, PH_NEWGAME = 3, PH_SOLVE = 4 /* waiting for the exact root solve */ };
constexpr uint8_t kSolveMarker = 0xFF;  // Descent::dihedral of a descent that waits for a WLD solve instead of a network evaluation

struct Slot {
    EnvState env;            // the real game
    u64 game_id;
    u64 games_played;        // games this slot has started
    uint32_t gen;            // hash generation tag of the current game (1..4095)
    uint32_t n_nodes, n_edges;
    uint32_t n_expand, n_rootsel, n_sims, sims_started, sims_target;
    uint32_t ply;            // decided plies recorded in the log so far
    uint8_t phase, tl, log_sel, enable_resign;
    uint8_t resigned_mask, search_only, n_pending, n_parked;
    uint8_t pending[kMaxK], parked[kMaxK];
    u64 root_own, root_enemy;
    uint8_t root_pid, black_net, white_net;  // black_net / white_net: networks of the two colours (matches, leagues)
    uint8_t root_req;         // 1: an exact root solve has to be put into this wave's solver batch
    uint8_t opening_plies;    // plies of the game's opening (rz_engine_set_openings), replayed before its first search
    uint32_t ply_waves;       // waves this slot has spent on the ply being decided (rz_ply::waves)
    uint32_t n_solves, n_searched_plies;
};

constexpr int kOpeningStride = RZ_MAX_OPENING_PLIES + 1;
constexpr int kCacheTurnBuckets = 61;  // turns 0..59 of the searched root; 60: the warm-started first game of a slot

struct Status {
    unsigned long long games_started, games_finished, expansions, simulations, plies, idle_slots;
    unsigned long long max_nodes, max_edges;
    int error;  // 0 or RZ_E*
    int pad;
    unsigned long long tower_rows, cache_repeats;
    unsigned long long cache_lookups[kCacheTurnBuckets], cache_hits[kCacheTurnBuckets];
};

struct DevCfg {
    int G, S, K, vl, change_tau_turn, thinking_loop, required_visit, start_rethinking_turn, allowed_resign_turn;
    int use_resign, share, max_plies, warm_start, sims_cap, n_nets, solver_turn, solver_sim_turn, keep_games;
    float c_puct, noise_eps, alpha, resign_threshold, disable_resignation_rate;
    u64 seed, first_game_id, game_id_stride, max_games;
    uint32_t nodes_cap, edges_cap, hash_cap;  // per slot (hash_cap is a power of two)
    float warm_cdf[60];  // warm_start: P(first game of a slot begins at turn <= t), rz_engine_set_warm_start_profile
    float warm_waves[60];  // ... and the waves a search at turn t takes in a long-running engine (0 = unknown)
};

__device__ __forceinline__ uint32_t hash_key(u64 own, u64 enemy, uint32_t kpid) {
    u64 h = own * 0x9E3779B97F4A7C15ULL ^ (enemy + 0x7F4A7C15ULL) * 0xC2B2AE3D27D4EB4FULL ^ (u64)kpid * 0x165667B19E3779F9ULL;
    h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ULL; h ^= h >> 32;
    return (uint32_t)h;
}

#include "rz_eval_cache.cuh"

struct DevPtrs {
    Slot* slots;
    Descent* desc;         // [G][K]
    uint32_t* hash;        // [G][hash_cap]
    Node* nodes;           // [G][nodes_cap]
    Edge* edges;           // [G][edges_cap]
    rz_ply* plies;         // [G][2][max_plies]
    rz_game* mail_hdr;     // [G][2]
    uint8_t* mail_flag;    // [G][2]  1 = finished game waiting for the host
    Status* status;
    uint32_t* batch_count; // leaves in the current batch: [group][net], 64 words apart
    u64* batch_own;        // [net][G*K] transformed, side-to-move frame
    u64* batch_enemy;
    float* policy;         // [net][G*K][64]
    float* value;          // [net][G*K]
    const uint8_t* net_table;  // [game][2]: networks of black and white (rz_engine_set_nets); NULL: alternate with the game
    const uint8_t* openings;   // [game][kOpeningStride]: number of plies, then the squares (rz_engine_set_openings); NULL: none
    // endgame solver: one resumable request context per descent (+ one per slot for the exact root solve), the lists of
    // unfinished requests (per group, double-buffered by wave parity) and the network results a waiting slot has to keep
    solver::SolveCtx* sctx;  // [G][K + 1]
    uint32_t* sactive;       // [2 groups][2 parities][G * (K + 1)]
    uint32_t* solve_count;   // [2 groups][2 parities] (64 words apart)
    float* keep_policy;      // [G*K][64]  (also where a leaf served by the evaluation cache finds its result)
    float* keep_value;       // [G*K]
    u64* solver_tt;          // per-lane transposition tables of the solver kernel, one set per slot group
    EvalCache cache;         // evaluation cache shared by both slot groups (n_sets == 0: off)
};

#include "rz_engine_warp.cuh"

// RZ_EVAL_FAKE: policy 1/64, value scale * (#own - #enemy)/64 (oracle/nn.py FakeNetAPI)
__global__ void fake_eval_kernel(const u64* __restrict__ own, const u64* __restrict__ enemy, const uint32_t* __restrict__ count,
                                 float* __restrict__ policy, float* __restrict__ value, float scale) {
    const uint32_t n = *count;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n * 64; i += gridDim.x * blockDim.x) {
        policy[i] = 1.0f / 64.0f;
        if ((i & 63) == 0) value[i >> 6] = scale * ((float)(popc64(own[i >> 6]) - popc64(enemy[i >> 6])) / 64.0f);
    }
}

__global__ void init_slots_kernel(const DevCfg c, const DevPtrs p) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= c.G) return;
    Slot& sl = p.slots[s];
    memset(&sl, 0, sizeof(Slot));
    sl.phase = PH_NEWGAME;
    p.mail_flag[(size_t)s * 2] = 0; p.mail_flag[(size_t)s * 2 + 1] = 0;
}

// single-position searches (rz_engine_search_root / rz_engine_search_roots): slot s < n_active searches roots[s], or roots[0]
// when there is one root, once (no game loop); the other slots go idle at once.  One warp per slot like the tick kernel.
// gid_stride: slot s draws the game id first_game_id + s * gid_stride (dihedral of each leaf evaluation, root noise).
struct Root { u64 own, enemy; uint32_t pid, pad; };

__global__ void setup_search_root_kernel(const DevCfg c, const DevPtrs p, const Root* __restrict__ roots, int n_roots, int n_active,
                                         u64 gid_stride, int keep_tree) {
    const int s = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (s >= c.G) return;
    if (s >= n_active) {
        if (lane == 0) { p.slots[s].phase = PH_IDLE; atomicAdd(&p.status->idle_slots, 1ULL); }
        return;
    }
    const Root r = roots[n_roots > 1 ? s : 0];
    const u64 own = r.own, enemy = r.enemy;
    const int pid = (int)r.pid;
    WCtx x(c, p, s, lane);
    Slot& sl = x.sl;
    sl.game_id = c.first_game_id + (u64)s * gid_stride;
    if (!keep_tree || sl.gen == 0) {
        sl.gen = sl.gen + 1;
        if (sl.gen >= 4096) {
            for (uint32_t i = lane; i < c.hash_cap; i += 32) x.hash[i] = 0;
            sl.gen = 1;
            __syncwarp();
        }
        sl.n_nodes = 0; sl.n_edges = 0; sl.n_expand = 0; sl.n_rootsel = 0; sl.n_sims = 0;
    }
    sl.ply = 0; sl.tl = 0;
    for (int k = 0; k < kMaxK; ++k) x.dstat[k] = k < c.K ? (uint8_t)D_FREE : (uint8_t)D_PENDING;
    env_update(sl.env, pid == 1 ? own : enemy, pid == 1 ? enemy : own, pid);
    x.begin_search(own, enemy, pid);
    sl.search_only = 1;
    x.write_back();
}
// root statistics of slots s0 .. s0 + gridDim.x - 1, one warp per slot, into rows 0 .. gridDim.x - 1 of n_out / w_out
__global__ void read_root_kernel(const DevCfg c, const DevPtrs p, int s0, int32_t* n_out, float* w_out) {
    WCtx x(c, p, s0 + (int)blockIdx.x, (int)threadIdx.x);
    n_out += (size_t)blockIdx.x * 64; w_out += (size_t)blockIdx.x * 64;
    n_out[threadIdx.x] = 0; n_out[threadIdx.x + 32] = 0; w_out[threadIdx.x] = 0.f; w_out[threadIdx.x + 32] = 0.f;
    __syncwarp();
    const int ni = x.find_node(x.sl.root_own, x.sl.root_enemy, x.kpid_of(x.sl.root_pid));
    if (ni < 0 || threadIdx.x != 0) return;
    const Node& nd = x.nodes[ni];
    u64 m = nd.legal;
    for (int i = 0; m; ++i, m &= m - 1) { n_out[ctz64(m)] = x.edges[nd.edge_base + i].n; w_out[ctz64(m)] = x.edges[nd.edge_base + i].w; }
}

}  // namespace eng
}  // namespace rz

using namespace rz;
using namespace rz::eng;

struct FinishedGame {
    rz_game hdr;
    std::vector<rz_ply> plies;
};

struct rz_engine {
    rz_engine_cfg cfg;
    DevCfg dc;
    DevPtrs dp;
    rz_net* net;                    // the network given at creation (self-play)
    rz_net* nets[RZ_MAX_NETS];      // the evaluators: nets[0] = net in self-play; matches and leagues set the list
    float fake_scale[RZ_MAX_NETS];  // RZ_EVAL_FAKE: value scale of each network
    int row_nets;                   // networks the row buffers and batch counters have room for
    uint8_t* d_net_table;           // rz_engine_set_nets: [game][2] on the device (NULL: none)
    uint64_t net_table_games;
    uint8_t* d_openings;            // rz_engine_set_openings: [game][kOpeningStride] on the device (NULL: none)
    uint64_t opening_games;
    int device;
    cudaStream_t stream;      // group 0 + all host<->device traffic
    cudaStream_t stream2;     // group 1 (tick of one group overlaps the network launch of the other)
    int n_groups;
    int group_slot0[3];
    size_t solver_tt_words_per_group;
    int solve_parity[2];      // per group: which of its two unfinished-solve lists the next wave reads
    long long solver_budget_ns;  // time the solver step may take per wave and group (RZ_SOLVER_BUDGET_US)
    void* arena[32];
    int n_arena;
    Status* h_status;     // pinned
    uint8_t* h_flags;     // pinned [G*2]
    uint64_t waves, nn_launches, mcts_launches;
    uint64_t finished_total;
    std::deque<FinishedGame> queue;  // producer: rz_engine_run (drain_mailboxes); consumer: rz_engine_poll, possibly on a second thread
    std::mutex queue_mutex;
    // device timing: 3 events per queued wave (before tick, between tick and evaluation, after evaluation)
    cudaEvent_t ev[2 * 3 * 8];  // [group][wave in burst][3]
    cudaEvent_t ev_run[3];     // run start, run end, group-1 join
    int ev_used;
    double nn_ms, mcts_ms, run_ms;
    uint32_t cache_sets;  // sets of the evaluation cache (0: off); dp.cache.n_sets is 0 while two networks play
    Root* d_roots;        // single-position searches: [G] roots, [G][64] root statistics (allocated on first use)
    int32_t* d_root_n;
    float* d_root_w;
};

constexpr int64_t kDefaultEvalCacheMb = 2048;

static int collect_timing(rz_engine* e) {  // call after the stream has been synchronised
    for (int g = 0; g < e->n_groups; ++g)
        for (int i = 0; i < e->ev_used; ++i) {
            float a = 0.f, b = 0.f;
            cudaEvent_t* ev = e->ev + (g * 8 + i) * 3;
            RZ_CUDA_TRY(cudaEventElapsedTime(&a, ev[0], ev[1]));
            RZ_CUDA_TRY(cudaEventElapsedTime(&b, ev[1], ev[2]));
            e->mcts_ms += a; e->nn_ms += b;
        }
    e->ev_used = 0;
    return RZ_OK;
}

static int dev_alloc(rz_engine* e, void** ptr, size_t bytes, bool zero) {
    if (e->n_arena >= (int)(sizeof(e->arena) / sizeof(e->arena[0]))) { set_error("rz_engine: allocation table full"); return RZ_ESTATE; }
    cudaError_t ce = cudaMalloc(ptr, bytes);
    if (ce != cudaSuccess) {
        set_error("rz_engine: cudaMalloc(%zu bytes) failed: %s", bytes, cudaGetErrorString(ce));
        cudaGetLastError();
        return RZ_ENOMEM;
    }
    e->arena[e->n_arena++] = *ptr;
    if (zero) RZ_CUDA_TRY(cudaMemsetAsync(*ptr, 0, bytes, e->stream));
    return RZ_OK;
}

// puts `fresh` in the place of *ptr in the allocation table (appends when *ptr is NULL) and frees the old buffer
static int arena_swap(rz_engine* e, void** ptr, void* fresh) {
    int i = 0;
    while (i < e->n_arena && (!*ptr || e->arena[i] != *ptr)) ++i;
    if (i == e->n_arena) {
        if (e->n_arena >= (int)(sizeof(e->arena) / sizeof(e->arena[0]))) { set_error("rz_engine: allocation table full"); return RZ_ESTATE; }
        e->n_arena++;
    }
    e->arena[i] = fresh;
    if (*ptr) RZ_CUDA_TRY(cudaFree(*ptr));
    *ptr = fresh;
    return RZ_OK;
}

// room for n_nets networks in the row buffers and batch counters (they only grow); on failure the old buffers stay
static int grow_rows(rz_engine* e, int n_nets) {
    if (n_nets <= e->row_nets) return RZ_OK;
    const size_t B = (size_t)n_nets * e->dc.G * e->dc.K;
    DevPtrs& p = e->dp;
    void** bufs[5] = {(void**)&p.batch_own, (void**)&p.batch_enemy, (void**)&p.policy, (void**)&p.value, (void**)&p.batch_count};
    const size_t bytes[5] = {(B + 2) * sizeof(u64), (B + 2) * sizeof(u64), (B + 2) * 64 * sizeof(float), (B + 2) * sizeof(float),
                             (size_t)n_nets * 2 * 64 * sizeof(uint32_t)};
    void* fresh[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    for (int i = 0; i < 5; ++i) {
        const cudaError_t ce = cudaMalloc(&fresh[i], bytes[i]);
        if (ce != cudaSuccess) {
            cudaGetLastError();
            for (int j = 0; j < i; ++j) cudaFree(fresh[j]);
            set_error("rz_engine: cudaMalloc(%zu bytes) for the rows of %d networks failed: %s", bytes[i], n_nets, cudaGetErrorString(ce));
            return RZ_ENOMEM;
        }
    }
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    for (int i = 0; i < 5; ++i) {
        RZ_CUDA_TRY(cudaMemsetAsync(fresh[i], 0, bytes[i], e->stream));
        RZ_TRY(arena_swap(e, bufs[i], fresh[i]));
    }
    e->row_nets = n_nets;
    return RZ_OK;
}

// the evaluators from the next wave on: n networks (1: self-play with the creation network), an optional game table
static void use_nets(rz_engine* e, rz_net* const* nets, const float* fake_scale, int n, const uint8_t* table) {
    for (int k = 0; k < RZ_MAX_NETS; ++k) {
        e->nets[k] = k < n && nets ? nets[k] : nullptr;
        e->fake_scale[k] = k < n && fake_scale ? fake_scale[k] : 1.f;
    }
    if (n == 1) e->nets[0] = e->net;
    e->dc.n_nets = n;
    e->dp.net_table = table;
    e->dp.cache.n_sets = n > 1 ? 0u : e->cache_sets;  // a leaf's result then depends on which network is to move
}

static int drain_mailboxes(rz_engine* e) {
    const int G = e->dc.G;
    RZ_CUDA_TRY(cudaMemcpyAsync(e->h_flags, e->dp.mail_flag, (size_t)G * 2, cudaMemcpyDeviceToHost, e->stream));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    for (int i = 0; i < G * 2; ++i) {
        if (!e->h_flags[i]) continue;
        FinishedGame fg;
        RZ_CUDA_TRY(cudaMemcpyAsync(&fg.hdr, e->dp.mail_hdr + i, sizeof(rz_game), cudaMemcpyDeviceToHost, e->stream));
        RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
        const int np = fg.hdr.n_plies;
        if (np < 0 || np > e->dc.max_plies) { set_error("rz_engine: corrupt mailbox (n_plies=%d)", np); return RZ_ESTATE; }
        fg.plies.resize((size_t)np);
        if (np) RZ_CUDA_TRY(cudaMemcpyAsync(fg.plies.data(), e->dp.plies + (size_t)i * e->dc.max_plies, (size_t)np * sizeof(rz_ply),
                                            cudaMemcpyDeviceToHost, e->stream));
        RZ_CUDA_TRY(cudaMemsetAsync(e->dp.mail_flag + i, 0, 1, e->stream));
        RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
        {
            std::lock_guard<std::mutex> lock(e->queue_mutex);
            e->queue.push_back(std::move(fg));
        }
        e->finished_total++;
    }
    return RZ_OK;
}

static int launch_wave(rz_engine* e) {
    const DevCfg& c = e->dc;
    const bool timed = e->ev_used < 8;
    if (e->dp.cache.n_sets) e->dp.cache.gen = (uint32_t)e->net->weights_version;  // new weights: every older entry misses
    for (int g = 0; g < e->n_groups; ++g) {
        cudaStream_t st = g == 0 ? e->stream : e->stream2;
        const int s0 = e->group_slot0[g], s1 = e->group_slot0[g + 1];
        cudaEvent_t* ev = e->ev + (g * 8 + e->ev_used) * 3;
        const size_t rows = (size_t)(s1 - s0) * c.K;
        if (timed) RZ_CUDA_TRY(cudaEventRecord(ev[0], st));
        RZ_CUDA_TRY(cudaMemsetAsync(e->dp.batch_count + g * c.n_nets * 64, 0, ((c.n_nets - 1) * 64 + 1) * sizeof(uint32_t), st));
        const bool solving = c.solver_turn > 0 || c.solver_sim_turn > 0;
        const int par = e->solve_parity[g];  // the unfinished-solve list this wave's tick appends to
        if (solving) RZ_CUDA_TRY(cudaMemsetAsync(e->dp.solve_count + (g * 2 + (1 - par)) * 64, 0, sizeof(uint32_t), st));
        tick_warp_kernel<<<(s1 - s0 + 1) / 2, kWarpTickThreads, 0, st>>>(c, e->dp, s0, s1, g, par);
        RZ_LAUNCH_CHECK();
        e->mcts_launches++;
        if (solving) {  // advance the group's unfinished solves for a bounded time (on the SMs the other group's tower leaves free)
            const size_t list = (size_t)c.G * (c.K + 1);
            solver::solve_active_kernel<<<num_sms(), solver::kBlockThreads, 0, st>>>(
                e->dp.sctx, e->dp.sactive + (g * 2 + par) * list, e->dp.solve_count + (g * 2 + par) * 64,
                e->dp.sactive + (g * 2 + (1 - par)) * list, e->dp.solve_count + (g * 2 + (1 - par)) * 64,
                e->dp.solver_tt + (size_t)g * e->solver_tt_words_per_group, e->solver_budget_ns);
            RZ_LAUNCH_CHECK();
            e->mcts_launches++;
            e->solve_parity[g] = 1 - par;
        }
        if (timed) RZ_CUDA_TRY(cudaEventRecord(ev[1], st));
        for (int net = 0; net < c.n_nets; ++net) {  // one evaluator launch per network, on that network's rows
            uint32_t* count = e->dp.batch_count + (g * c.n_nets + net) * 64;
            const size_t row0 = (size_t)net * c.G * c.K + (size_t)s0 * c.K;
            if (e->cfg.eval_mode == RZ_EVAL_FAKE) {
                fake_eval_kernel<<<num_sms() * 4, 256, 0, st>>>(e->dp.batch_own + row0, e->dp.batch_enemy + row0, count, e->dp.policy + row0 * 64,
                                                              e->dp.value + row0, e->fake_scale[net]);
                RZ_LAUNCH_CHECK();
                e->mcts_launches++;
            } else {
                RZ_TRY(net_forward(e->nets[net], e->dp.batch_own + row0, e->dp.batch_enemy + row0, e->dp.policy + row0 * 64,
                                   e->dp.value + row0, rows, count, e->cfg.net_impl, st, nullptr));
                e->nn_launches++;
            }
        }
        if (timed) RZ_CUDA_TRY(cudaEventRecord(ev[2], st));
        if (e->dp.cache.n_sets) {  // this wave's tower rows into the evaluation cache (outside the timed evaluation)
            cache_insert_kernel<<<num_sms() * 2, 256, 0, st>>>(e->dp.cache, e->dp.batch_own + (size_t)s0 * c.K, e->dp.batch_enemy + (size_t)s0 * c.K,
                                                              e->dp.policy + (size_t)s0 * c.K * 64, e->dp.value + (size_t)s0 * c.K,
                                                              e->dp.batch_count + g * c.n_nets * 64, &e->dp.status->cache_repeats);
            RZ_LAUNCH_CHECK();
            e->mcts_launches++;
        }
    }
    if (timed) e->ev_used++;
    e->waves++;
    return RZ_OK;
}

static int sync_all(rz_engine* e) {
    if (e->n_groups > 1) RZ_CUDA_TRY(cudaStreamSynchronize(e->stream2));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return RZ_OK;
}

static int read_status(rz_engine* e) {
    RZ_TRY(sync_all(e));
    RZ_CUDA_TRY(cudaMemcpyAsync(e->h_status, e->dp.status, sizeof(Status), cudaMemcpyDeviceToHost, e->stream));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    RZ_TRY(collect_timing(e));
    if (e->h_status->error != 0) {
        set_error("rz_engine: device-side failure %d (%s)", e->h_status->error,
                  e->h_status->error == RZ_ECAPACITY ? "node/edge/ply arena overflow" : "inconsistent search state");
        return e->h_status->error;
    }
    return RZ_OK;
}

// Single-position searches: slots 0 .. n_active - 1 search their roots (see setup_search_root_kernel), then the root
// statistics of slots read0 .. read0 + n_read - 1 come back in one readout launch and one copy per array.
static int search_slots(rz_engine* e, const Root* roots, int n_roots, int n_active, u64 gid_stride, int keep_tree, int read0,
                        int n_read, int32_t* n_visit, float* w_sum) {
    const size_t G = (size_t)e->dc.G;
    RZ_CUDA_TRY(cudaSetDevice(e->device));
    RZ_TRY(sync_all(e));
    if (!e->d_roots) {
        RZ_TRY(dev_alloc(e, (void**)&e->d_roots, G * sizeof(Root), false));
        RZ_TRY(dev_alloc(e, (void**)&e->d_root_n, G * 64 * sizeof(int32_t), false));
        RZ_TRY(dev_alloc(e, (void**)&e->d_root_w, G * 64 * sizeof(float), false));
    }
    RZ_CUDA_TRY(cudaMemcpyAsync(e->d_roots, roots, (size_t)n_roots * sizeof(Root), cudaMemcpyHostToDevice, e->stream));
    RZ_CUDA_TRY(cudaMemsetAsync(e->dp.status, 0, sizeof(Status), e->stream));
    setup_search_root_kernel<<<(e->dc.G + 3) / 4, 128, 0, e->stream>>>(e->dc, e->dp, e->d_roots, n_roots, n_active, gid_stride, keep_tree);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    for (int it = 0; it < 1000000; ++it) {
        for (int i = 0; i < 8; ++i) RZ_TRY(launch_wave(e));
        RZ_TRY(read_status(e));
        if (e->h_status->idle_slots >= (unsigned long long)e->dc.G) break;
    }
    read_root_kernel<<<n_read, 32, 0, e->stream>>>(e->dc, e->dp, read0, e->d_root_n, e->d_root_w);
    RZ_LAUNCH_CHECK();
    RZ_CUDA_TRY(cudaMemcpyAsync(n_visit, e->d_root_n, (size_t)n_read * 64 * sizeof(int32_t), cudaMemcpyDeviceToHost, e->stream));
    RZ_CUDA_TRY(cudaMemcpyAsync(w_sum, e->d_root_w, (size_t)n_read * 64 * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    return RZ_OK;
}

extern "C" {

int rz_engine_create(const rz_engine_cfg* cfg, rz_net* net, int device, rz_engine** out) {
    RZ_REQUIRE(cfg && out, "rz_engine_create: null pointer");
    RZ_REQUIRE(cfg->games >= 1 && cfg->games <= (1 << 20), "games out of range (%d)", cfg->games);
    RZ_REQUIRE(cfg->simulation_num_per_move >= 1 && cfg->simulation_num_per_move <= 100000, "simulation_num_per_move out of range");
    RZ_REQUIRE(cfg->parallel_search_num >= 1 && cfg->parallel_search_num <= kMaxK, "parallel_search_num must be 1..%d", kMaxK);
    RZ_REQUIRE(cfg->thinking_loop >= 1 && cfg->thinking_loop <= 255, "thinking_loop must be 1..255");
    RZ_REQUIRE(cfg->eval_mode == RZ_EVAL_FAKE || net, "rz_engine_create: a network is required unless eval_mode == RZ_EVAL_FAKE");
    RZ_REQUIRE(cfg->game_id_stride >= 1, "game_id_stride must be >= 1");
    RZ_CUDA_TRY(cudaSetDevice(device));
    rz_engine* e = new (std::nothrow) rz_engine();
    if (!e) { set_error("out of host memory"); return RZ_ENOMEM; }
    e->cfg = *cfg; e->net = net; e->device = device; e->n_arena = 0;
    for (int k = 0; k < RZ_MAX_NETS; ++k) { e->nets[k] = nullptr; e->fake_scale[k] = 1.f; }
    e->nets[0] = net;
    e->row_nets = 2;
    e->d_net_table = nullptr; e->net_table_games = 0;
    e->d_openings = nullptr; e->opening_games = 0;
    e->waves = e->nn_launches = e->mcts_launches = e->finished_total = 0;
    e->h_status = nullptr; e->h_flags = nullptr; e->stream = nullptr; e->stream2 = nullptr;
    e->ev_used = 0; e->nn_ms = e->mcts_ms = e->run_ms = 0.0;
    e->cache_sets = 0;
    e->d_roots = nullptr; e->d_root_n = nullptr; e->d_root_w = nullptr;
    for (int i = 0; i < 48; ++i) e->ev[i] = nullptr;
    e->ev_run[0] = e->ev_run[1] = e->ev_run[2] = nullptr;
    // two slot groups on two streams: the MCTS tick of one group can run while the network launch of the other is in flight,
    // on the SMs that launch leaves free (a tower CTA takes nearly all of an SM's registers), or right after it
    e->n_groups = cfg->overlap_groups == 1 ? 1 : (cfg->overlap_groups == 2 ? 2 : (cfg->games >= 256 ? 2 : 1));
    if (cfg->games < 2) e->n_groups = 1;
    e->group_slot0[0] = 0;
    e->group_slot0[1] = e->n_groups == 2 ? (cfg->games + 1) / 2 : cfg->games;
    e->group_slot0[2] = cfg->games;
    DevCfg& c = e->dc;
    c.G = cfg->games; c.S = cfg->simulation_num_per_move; c.K = cfg->parallel_search_num; c.vl = cfg->virtual_loss;
    c.change_tau_turn = cfg->change_tau_turn; c.thinking_loop = cfg->thinking_loop; c.required_visit = cfg->required_visit_to_decide_action;
    c.start_rethinking_turn = cfg->start_rethinking_turn; c.allowed_resign_turn = cfg->allowed_resign_turn;
    c.use_resign = cfg->use_resign_threshold; c.share = cfg->share_mtcs_info; c.max_plies = cfg->max_plies > 0 ? cfg->max_plies : 64;
    c.warm_start = cfg->warm_start;
    for (int t = 0; t < 60; ++t) { c.warm_cdf[t] = t < 58 ? (float)(t + 1) / 58.f : 1.f; c.warm_waves[t] = 0.f; }  // default: turns 0..57 equally likely
    c.n_nets = 1;
    c.keep_games = cfg->reset_mtcs_info_per_game > 1 ? cfg->reset_mtcs_info_per_game : 1;
    c.solver_turn = cfg->use_solver_turn; c.solver_sim_turn = cfg->use_solver_turn_in_simulation;
    c.sims_cap = cfg->max_sims_per_wave > 0 ? cfg->max_sims_per_wave : 2 * cfg->parallel_search_num;
    c.c_puct = cfg->c_puct; c.noise_eps = cfg->noise_eps; c.alpha = cfg->dirichlet_alpha; c.resign_threshold = cfg->resign_threshold;
    c.disable_resignation_rate = cfg->disable_resignation_rate;
    c.seed = cfg->seed; c.first_game_id = cfg->first_game_id; c.game_id_stride = cfg->game_id_stride; c.max_games = cfg->max_games;
    // every simulation creates at most one node; a game has at most 60 searched plies
    const uint64_t searches = cfg->max_searches_per_game > 0 ? (uint64_t)cfg->max_searches_per_game
                                                              : (uint64_t)60 * (c.thinking_loop > 2 ? 2 : c.thinking_loop);
    const uint64_t arena_sims = cfg->arena_simulation_num > c.S ? (uint64_t)cfg->arena_simulation_num : (uint64_t)c.S;
    uint64_t nodes = searches * arena_sims * (uint64_t)c.keep_games + 64;
    if (nodes > 0xFFFF0) nodes = 0xFFFF0;
    c.nodes_cap = (uint32_t)nodes;
    c.edges_cap = c.nodes_cap * 14;
    uint32_t h = 1024;
    while (h < 2 * c.nodes_cap) h <<= 1;
    c.hash_cap = h;
    int rc = RZ_OK;
    cudaError_t ce = cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking);
    if (ce == cudaSuccess) ce = cudaStreamCreateWithFlags(&e->stream2, cudaStreamNonBlocking);
    if (ce != cudaSuccess) { set_error("cudaStreamCreate: %s", cudaGetErrorString(ce)); delete e; return RZ_ECUDA; }
    const size_t G = c.G, B = (size_t)e->row_nets * G * c.K;  // rows for two networks (evaluation matches); self-play uses the first part
    DevPtrs& p = e->dp;
    rc = dev_alloc(e, (void**)&p.slots, G * sizeof(Slot), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.desc, G * c.K * sizeof(Descent), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.hash, G * c.hash_cap * sizeof(uint32_t), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.nodes, G * c.nodes_cap * sizeof(Node), false);
    if (!rc) rc = dev_alloc(e, (void**)&p.edges, G * (size_t)c.edges_cap * sizeof(Edge), false);
    if (!rc) rc = dev_alloc(e, (void**)&p.plies, G * 2 * c.max_plies * sizeof(rz_ply), false);
    if (!rc) rc = dev_alloc(e, (void**)&p.mail_hdr, G * 2 * sizeof(rz_game), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.mail_flag, G * 2, true);
    if (!rc) rc = dev_alloc(e, (void**)&p.status, sizeof(Status), true);
    p.net_table = nullptr;
    p.openings = nullptr;
    if (!rc) rc = dev_alloc(e, (void**)&p.batch_count, (size_t)e->row_nets * 2 * 64 * sizeof(uint32_t), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.batch_own, (B + 2) * sizeof(u64), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.batch_enemy, (B + 2) * sizeof(u64), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.policy, (B + 2) * 64 * sizeof(float), true);
    if (!rc) rc = dev_alloc(e, (void**)&p.value, (B + 2) * sizeof(float), true);
    const bool solving = c.solver_turn > 0 || c.solver_sim_turn > 0;
    const size_t SR = G * (c.K + 1);
    // evaluation cache: on by default for the network evaluator (RZ_EVAL_CACHE_MB overrides the default size)
    int64_t cache_mb = cfg->eval_cache_mb;
    if (cache_mb == 0) {
        const char* env = getenv("RZ_EVAL_CACHE_MB");
        cache_mb = env ? atoll(env) : kDefaultEvalCacheMb;
    }
    if (cfg->eval_mode != RZ_EVAL_NET) cache_mb = 0;
    const size_t cache_sets = cache_mb > 0 ? (size_t)cache_mb * 1048576 / (kCacheWays * sizeof(EvalCacheEntry)) : 0;
    p.cache.entries = nullptr; p.cache.next = nullptr; p.cache.n_sets = 0; p.cache.gen = 0;
    if (!rc && cache_sets >= 0xFFFFFFFFull / kCacheWays) { set_error("eval_cache_mb too large (%lld)", (long long)cache_mb); rc = RZ_EINVAL; }
    if (!rc && cache_sets) {
        if (!rc) rc = dev_alloc(e, (void**)&p.cache.entries, cache_sets * kCacheWays * sizeof(EvalCacheEntry), true);
        if (!rc) rc = dev_alloc(e, (void**)&p.cache.next, cache_sets * sizeof(uint32_t), true);
        e->cache_sets = (uint32_t)cache_sets;
        p.cache.n_sets = e->cache_sets;
    }
    if (!rc) rc = dev_alloc(e, (void**)&p.solve_count, 1024, true);
    p.sctx = nullptr; p.sactive = nullptr; p.keep_policy = nullptr; p.keep_value = nullptr; p.solver_tt = nullptr;
    e->solve_parity[0] = e->solve_parity[1] = 0;
    {
        const char* b = getenv("RZ_SOLVER_BUDGET_US");
        const long long us = b ? atoll(b) : 2000;
        e->solver_budget_ns = (us > 0 ? us : 2000) * 1000LL;
    }
    // one transposition table per lane of the solver step's grid (one CTA per SM), one set per slot group
    e->solver_tt_words_per_group = (size_t)num_sms() * solver::kBlockThreads * solver::kTtEntries * solver::kTtWordsPerEntry;
    if (solving) {
        if (!rc) rc = dev_alloc(e, (void**)&p.sctx, SR * sizeof(solver::SolveCtx), true);
        if (!rc) rc = dev_alloc(e, (void**)&p.sactive, 4 * SR * sizeof(uint32_t), true);
        if (!rc) rc = dev_alloc(e, (void**)&p.solver_tt, e->solver_tt_words_per_group * 2 * sizeof(u64), true);
    }
    if (solving || cache_sets) {
        if (!rc) rc = dev_alloc(e, (void**)&p.keep_policy, G * c.K * 64 * sizeof(float), true);
        if (!rc) rc = dev_alloc(e, (void**)&p.keep_value, G * c.K * sizeof(float), true);
    }
    if (!rc && cudaMallocHost((void**)&e->h_status, sizeof(Status)) != cudaSuccess) { set_error("cudaMallocHost failed"); rc = RZ_ENOMEM; }
    if (!rc && cudaMallocHost((void**)&e->h_flags, G * 2) != cudaSuccess) { set_error("cudaMallocHost failed"); rc = RZ_ENOMEM; }
    for (int i = 0; i < 48 && !rc; ++i)
        if (cudaEventCreate(&e->ev[i]) != cudaSuccess) { set_error("cudaEventCreate failed"); rc = RZ_ECUDA; }
    for (int i = 0; i < 3 && !rc; ++i)
        if (cudaEventCreate(&e->ev_run[i]) != cudaSuccess) { set_error("cudaEventCreate failed"); rc = RZ_ECUDA; }
    if (rc) { rz_engine_destroy(e); return rc; }
    init_slots_kernel<<<(c.G + 127) / 128, 128, 0, e->stream>>>(c, p);
    ce = cudaStreamSynchronize(e->stream);
    if (ce != cudaSuccess) { set_error("rz_engine_create: %s", cudaGetErrorString(ce)); rz_engine_destroy(e); return RZ_ECUDA; }
    *out = e;
    return RZ_OK;
}

int rz_engine_destroy(rz_engine* e) {
    if (!e) return RZ_OK;
    cudaSetDevice(e->device);
    if (e->stream2) cudaStreamSynchronize(e->stream2);
    if (e->stream) cudaStreamSynchronize(e->stream);
    for (int i = 0; i < e->n_arena; ++i) cudaFree(e->arena[i]);
    if (e->h_status) cudaFreeHost(e->h_status);
    if (e->h_flags) cudaFreeHost(e->h_flags);
    for (int i = 0; i < 48; ++i) if (e->ev[i]) cudaEventDestroy(e->ev[i]);
    for (int i = 0; i < 3; ++i) if (e->ev_run[i]) cudaEventDestroy(e->ev_run[i]);
    if (e->stream) cudaStreamDestroy(e->stream);
    if (e->stream2) cudaStreamDestroy(e->stream2);
    cudaGetLastError();
    delete e;
    return RZ_OK;
}

int rz_engine_run(rz_engine* e, uint64_t finished_target, uint64_t max_waves) {
    RZ_REQUIRE(e, "rz_engine_run: null engine");
    RZ_CUDA_TRY(cudaSetDevice(e->device));
    const uint64_t wave0 = e->waves;
    const int kCheck = 8;  // waves queued between host checks
    RZ_TRY(sync_all(e));
    RZ_CUDA_TRY(cudaEventRecord(e->ev_run[0], e->stream));
    if (e->n_groups > 1) RZ_CUDA_TRY(cudaStreamWaitEvent(e->stream2, e->ev_run[0], 0));
    int rc_loop = RZ_OK;
    while (true) {
        if (e->finished_total >= finished_target && finished_target > 0) break;
        if (max_waves && e->waves - wave0 >= max_waves) break;
        int burst = kCheck;
        if (max_waves && e->waves - wave0 + burst > max_waves) burst = (int)(max_waves - (e->waves - wave0));
        for (int i = 0; i < burst; ++i) RZ_TRY(launch_wave(e));
        RZ_TRY(read_status(e));
        if (e->h_status->games_finished > e->finished_total) RZ_TRY(drain_mailboxes(e));
        if (e->h_status->idle_slots >= (unsigned long long)e->dc.G) {  // every slot ran out of games
            RZ_TRY(drain_mailboxes(e));
            break;
        }
    }
    (void)rc_loop;
    if (e->n_groups > 1) {
        RZ_CUDA_TRY(cudaEventRecord(e->ev_run[2], e->stream2));
        RZ_CUDA_TRY(cudaStreamWaitEvent(e->stream, e->ev_run[2], 0));
    }
    RZ_CUDA_TRY(cudaEventRecord(e->ev_run[1], e->stream));
    RZ_TRY(sync_all(e));
    float ms = 0.f;
    RZ_CUDA_TRY(cudaEventElapsedTime(&ms, e->ev_run[0], e->ev_run[1]));
    e->run_ms += ms;
    return RZ_OK;
}

int rz_engine_poll(rz_engine* e, rz_game* games, size_t game_cap, size_t* n_games, rz_ply* plies, size_t ply_cap, size_t* n_plies) {
    RZ_REQUIRE(e && n_games && n_plies, "rz_engine_poll: null pointer");
    size_t ng = 0, np = 0;
    std::lock_guard<std::mutex> lock(e->queue_mutex);
    while (!e->queue.empty() && ng < game_cap) {
        FinishedGame& fg = e->queue.front();
        if (np + fg.plies.size() > ply_cap) break;
        games[ng] = fg.hdr;
        games[ng].first_ply = (int32_t)np;
        if (!fg.plies.empty()) memcpy(plies + np, fg.plies.data(), fg.plies.size() * sizeof(rz_ply));
        np += fg.plies.size();
        ++ng;
        e->queue.pop_front();
    }
    *n_games = ng; *n_plies = np;
    return RZ_OK;
}

int rz_engine_stats(rz_engine* e, rz_stats* out) {
    RZ_REQUIRE(e && out, "rz_engine_stats: null pointer");
    RZ_CUDA_TRY(cudaSetDevice(e->device));
    RZ_TRY(sync_all(e));
    RZ_CUDA_TRY(cudaMemcpyAsync(e->h_status, e->dp.status, sizeof(Status), cudaMemcpyDeviceToHost, e->stream));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    const Status& s = *e->h_status;
    out->games_started = s.games_started; out->games_finished = s.games_finished; out->expansions = s.expansions;
    out->simulations = s.simulations; out->waves = e->waves; out->plies = s.plies; out->nn_launches = e->nn_launches;
    out->mcts_launches = e->mcts_launches; out->max_nodes_used = s.max_nodes; out->max_edges_used = s.max_edges;
    RZ_TRY(collect_timing(e));
    out->nn_ms = e->nn_ms; out->mcts_ms = e->mcts_ms; out->run_ms = e->run_ms;
    out->tower_rows = s.tower_rows; out->cache_repeats = s.cache_repeats;
    out->cache_lookups = out->cache_hits = 0;
    for (int b = 0; b < kCacheTurnBuckets; ++b) { out->cache_lookups += s.cache_lookups[b]; out->cache_hits += s.cache_hits[b]; }
    return RZ_OK;
}

int rz_engine_cache_turn_stats(rz_engine* e, uint64_t* lookups, uint64_t* hits, int n) {
    RZ_REQUIRE(e && lookups && hits && n == kCacheTurnBuckets, "rz_engine_cache_turn_stats: bad argument");
    RZ_CUDA_TRY(cudaSetDevice(e->device));
    RZ_TRY(sync_all(e));
    RZ_CUDA_TRY(cudaMemcpyAsync(e->h_status, e->dp.status, sizeof(Status), cudaMemcpyDeviceToHost, e->stream));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    for (int b = 0; b < n; ++b) { lookups[b] = e->h_status->cache_lookups[b]; hits[b] = e->h_status->cache_hits[b]; }
    return RZ_OK;
}

int rz_engine_set_simulation_num(rz_engine* e, int32_t sims) {
    RZ_REQUIRE(e && sims >= 1, "rz_engine_set_simulation_num: bad argument");
    const uint64_t searches = e->cfg.max_searches_per_game > 0 ? (uint64_t)e->cfg.max_searches_per_game
                                                                  : (uint64_t)60 * (e->dc.thinking_loop > 2 ? 2 : e->dc.thinking_loop);
    uint64_t need = searches * sims * (uint64_t)e->dc.keep_games + 64;
    RZ_REQUIRE(need <= e->dc.nodes_cap, "simulation count %d exceeds the arenas sized at creation", sims);
    e->dc.S = sims;
    e->cfg.simulation_num_per_move = sims;
    return RZ_OK;
}

int rz_engine_set_max_games(rz_engine* e, uint64_t max_games) {
    RZ_REQUIRE(e, "rz_engine_set_max_games: null engine");
    RZ_REQUIRE(!e->dp.net_table || (max_games >= 1 && max_games <= e->net_table_games),
               "rz_engine_set_max_games: %llu games with a network table of %llu games", (unsigned long long)max_games,
               (unsigned long long)e->net_table_games);
    RZ_REQUIRE(!e->dp.openings || (max_games >= 1 && max_games <= e->opening_games),
               "rz_engine_set_max_games: %llu games with an opening table of %llu games", (unsigned long long)max_games,
               (unsigned long long)e->opening_games);
    e->dc.max_games = max_games;
    e->cfg.max_games = max_games;
    return RZ_OK;
}

int rz_engine_set_warm_start_profile(rz_engine* e, const float* weight, int n) {
    RZ_REQUIRE(e && weight && n >= 1 && n <= 60, "rz_engine_set_warm_start_profile: bad argument");
    RZ_REQUIRE(e->waves == 0, "rz_engine_set_warm_start_profile: must be called before the first wave");
    double total = 0.0;
    for (int t = 0; t < n; ++t) {
        RZ_REQUIRE(weight[t] >= 0.f, "rz_engine_set_warm_start_profile: negative weight");
        total += weight[t];
    }
    RZ_REQUIRE(total > 0.0, "rz_engine_set_warm_start_profile: all weights are zero");
    double cum = 0.0;
    for (int t = 0; t < 60; ++t) {
        if (t < n) cum += weight[t];
        e->dc.warm_cdf[t] = t >= n - 1 ? 1.f : (float)(cum / total);
        e->dc.warm_waves[t] = t < n ? weight[t] : 0.f;
    }
    return RZ_OK;
}

int rz_engine_set_second_net(rz_engine* e, rz_net* net_b, int enable) {
    RZ_REQUIRE(e, "rz_engine_set_second_net: null engine");
    RZ_REQUIRE(!enable || e->cfg.eval_mode == RZ_EVAL_FAKE || net_b, "rz_engine_set_second_net: a second network is required");
    RZ_REQUIRE(e->waves == 0, "rz_engine_set_second_net: must be called before the first wave");
    rz_net* const nets[2] = {e->net, net_b};
    const float scale[2] = {1.f, -1.f};
    use_nets(e, nets, scale, enable ? 2 : 1, nullptr);
    return RZ_OK;
}

int rz_engine_set_nets(rz_engine* e, rz_net* const* nets, const float* fake_scale, int n_nets, const uint8_t* black_net,
                       const uint8_t* white_net, uint64_t n_games) {
    RZ_REQUIRE(e && black_net && white_net, "rz_engine_set_nets: null pointer");
    RZ_REQUIRE(e->waves == 0, "rz_engine_set_nets: must be called before the first wave");
    RZ_REQUIRE(n_nets >= 2 && n_nets <= RZ_MAX_NETS, "rz_engine_set_nets: n_nets = %d outside 2..%d", n_nets, RZ_MAX_NETS);
    if (e->cfg.eval_mode == RZ_EVAL_NET) {
        RZ_REQUIRE(nets, "rz_engine_set_nets: networks are required unless eval_mode == RZ_EVAL_FAKE");
        for (int k = 0; k < n_nets; ++k) RZ_REQUIRE(nets[k], "rz_engine_set_nets: network %d is NULL", k);
    }
    RZ_REQUIRE(e->dc.max_games >= 1 && e->dc.max_games <= n_games,
               "rz_engine_set_nets: max_games = %llu must be 1..n_games (%llu): the table has no entry for later games",
               (unsigned long long)e->dc.max_games, (unsigned long long)n_games);
    std::vector<uint8_t> table((size_t)n_games * 2);
    for (uint64_t i = 0; i < n_games; ++i) {
        RZ_REQUIRE(black_net[i] < n_nets && white_net[i] < n_nets, "rz_engine_set_nets: game %llu: networks %d / %d, but n_nets = %d",
                   (unsigned long long)i, (int)black_net[i], (int)white_net[i], n_nets);
        table[2 * i] = black_net[i];
        table[2 * i + 1] = white_net[i];
    }
    RZ_CUDA_TRY(cudaSetDevice(e->device));
    uint8_t* d_table = nullptr;
    if (cudaMalloc((void**)&d_table, table.size()) != cudaSuccess) {
        cudaGetLastError();
        set_error("rz_engine_set_nets: cudaMalloc(%zu bytes) failed", table.size());
        return RZ_ENOMEM;
    }
    int rc = grow_rows(e, n_nets);
    if (rc) { cudaFree(d_table); return rc; }
    RZ_CUDA_TRY(cudaMemcpyAsync(d_table, table.data(), table.size(), cudaMemcpyHostToDevice, e->stream));
    RZ_CUDA_TRY(cudaStreamSynchronize(e->stream));
    RZ_TRY(arena_swap(e, (void**)&e->d_net_table, d_table));
    e->net_table_games = n_games;
    use_nets(e, nets, fake_scale, n_nets, e->d_net_table);
    return RZ_OK;
}

int rz_engine_set_openings(rz_engine* e, const uint8_t* moves, const uint8_t* n_moves, uint64_t n_games) {
    RZ_REQUIRE(e && moves && n_moves, "rz_engine_set_openings: null pointer");
    RZ_REQUIRE(e->waves == 0, "rz_engine_set_openings: must be called before the first wave");
    RZ_REQUIRE(!e->dc.warm_start, "rz_engine_set_openings: warm_start already chooses where the first games begin");
    RZ_REQUIRE(e->dc.max_games >= 1 && e->dc.max_games <= n_games,
               "rz_engine_set_openings: max_games = %llu must be 1..n_games (%llu): the table has no entry for later games",
               (unsigned long long)e->dc.max_games, (unsigned long long)n_games);
    std::vector<uint8_t> table((size_t)n_games * kOpeningStride, 0);
    for (uint64_t i = 0; i < n_games; ++i) {
        const int n = n_moves[i];
        RZ_REQUIRE(n <= RZ_MAX_OPENING_PLIES, "rz_engine_set_openings: game %llu: %d moves, at most %d", (unsigned long long)i, n,
                   RZ_MAX_OPENING_PLIES);
        // the env would end a game at an illegal move; an opening must be legal, and never pass or finish the game
        EnvState env;
        env_reset(env);
        for (int j = 0; j < n; ++j) {
            const int mv = moves[i * RZ_MAX_OPENING_PLIES + j];
            const bool b = env.next_player == 1;
            const u64 legal = mv < 64 ? find_correct_moves(b ? env.black : env.white, b ? env.white : env.black) : 0;
            RZ_REQUIRE((legal >> mv) & 1, "rz_engine_set_openings: game %llu: move %d (square %d) is illegal", (unsigned long long)i, j + 1, mv);
            const uint8_t mover = env.next_player;
            env_step(env, mv);
            RZ_REQUIRE(!env.done, "rz_engine_set_openings: game %llu: move %d ends the game", (unsigned long long)i, j + 1);
            RZ_REQUIRE(env.next_player != mover, "rz_engine_set_openings: game %llu: after move %d the other side must pass",
                       (unsigned long long)i, j + 1);
            table[(size_t)i * kOpeningStride + 1 + j] = (uint8_t)mv;
        }
        table[(size_t)i * kOpeningStride] = (uint8_t)n;
    }
    RZ_CUDA_TRY(cudaSetDevice(e->device));
    uint8_t* d_table = nullptr;
    if (cudaMalloc((void**)&d_table, table.size()) != cudaSuccess) {
        cudaGetLastError();
        set_error("rz_engine_set_openings: cudaMalloc(%zu bytes) failed", table.size());
        return RZ_ENOMEM;
    }
    const cudaError_t ce = cudaMemcpy(d_table, table.data(), table.size(), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) {
        cudaFree(d_table);
        set_error("rz_engine_set_openings: cudaMemcpy: %s", cudaGetErrorString(ce));
        return RZ_ECUDA;
    }
    RZ_TRY(arena_swap(e, (void**)&e->d_openings, d_table));
    e->opening_games = n_games;
    e->dp.openings = e->d_openings;
    return RZ_OK;
}

int rz_engine_set_resign_threshold(rz_engine* e, int use_resign_threshold, float resign_threshold) {
    RZ_REQUIRE(e, "rz_engine_set_resign_threshold: null engine");
    e->dc.use_resign = use_resign_threshold ? 1 : 0;
    e->dc.resign_threshold = resign_threshold;
    e->cfg.use_resign_threshold = e->dc.use_resign;
    e->cfg.resign_threshold = resign_threshold;
    return RZ_OK;
}

int rz_engine_search_root(rz_engine* e, uint64_t own, uint64_t enemy, int player, int slot, int keep_tree, int32_t* n_visit,
                          float* w_sum) {
    RZ_REQUIRE(e && n_visit && w_sum && (player == 1 || player == 2) && slot >= 0 && slot < e->dc.G, "rz_engine_search_root: bad argument");
    const Root r{own, enemy, (uint32_t)player, 0};
    return search_slots(e, &r, 1, e->dc.G, e->dc.game_id_stride, keep_tree, slot, 1, n_visit, w_sum);
}

int rz_engine_search_roots(rz_engine* e, const uint64_t* own, const uint64_t* enemy, const uint8_t* player, int n, int keep_tree,
                           int32_t* n_visit, float* w_sum) {
    RZ_REQUIRE(e && own && enemy && player && n_visit && w_sum, "rz_engine_search_roots: null pointer");
    RZ_REQUIRE(n >= 1 && n <= e->dc.G, "rz_engine_search_roots: n = %d outside 1..%d (the engine's slots)", n, e->dc.G);
    std::vector<Root> roots((size_t)n);
    for (int i = 0; i < n; ++i) {
        RZ_REQUIRE(player[i] == 1 || player[i] == 2, "rz_engine_search_roots: player[%d] = %d is not 1 or 2", i, (int)player[i]);
        RZ_REQUIRE(find_correct_moves(own[i], enemy[i]) != 0, "rz_engine_search_roots: root %d has no legal move for its mover", i);
        roots[(size_t)i] = Root{own[i], enemy[i], (uint32_t)player[i], 0};
    }
    // With root noise off the game id only picks the dihedral of each leaf evaluation: every slot then uses the first game
    // id, so that a position gives the same statistics whatever slot it is searched in (those of a one-slot engine).
    const u64 gid_stride = e->dc.noise_eps > 0.f ? e->dc.game_id_stride : 0;
    return search_slots(e, roots.data(), n, n, gid_stride, keep_tree, 0, n, n_visit, w_sum);
}

}  // extern "C"
